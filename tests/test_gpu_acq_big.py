"""LogEI, LogPoI, MES and the constrained acquisitions (DESIGN.md 4.10 - 4.12), values and input gradients, at
production sizes on ill-conditioned training sets, against a double-double reference.

The fixtures (oracle/make_acq_big.py, tests/golden/acqbig_*.npz) hold the 50-digit values of every kind, evaluated on
the unrounded double-double mu and sigma^2, on the four problems of tests/test_gpu_illcond_big.py (N = 1000 .. 4096,
cond(K) 6.5e6 .. 1.8e11) and at bench.py's C5 shape (b_m25_c5: N = 8192, d = 32, cond(K) 2.8e9), with two constraint
GPs on b_m15_d17 (np = 1024) and b_m25_c3 (np = 4096), and their input gradients on 64 rows.  The referee is sklearn's
fp64 mu and sigma through tests/logei_oracle.py / tests/mes_oracle.py, and tests/grad_oracle.py's Cholesky solves for
the gradients.

The rules are those of tests/test_gpu_illcond.py: device error <= max(C_REF * the referee's error, FLOOR) with
C_REF = 100 (every value here derives from sigma), the 1e-5 bar wherever the referee meets it, and per-problem bars
pinned at about 10x the error measured on an H100 80GB HBM3 at a 700 W power limit (in the comments).  Metrics: LogEI
and LogPoI |d| / (1 + |v|); MES, UCB / EI / PoI and the product forms relative to the batch's largest |value|;
gradients max_j |d g_j| / (max_j |g_j| + |value| / l_min + 1e-6) per row (DESIGN.md 4.10).  Every case prints the
device's and the referee's errors (pytest -s).  The module takes about 35 s on that GPU (measured 34 s).
"""
import ctypes as C
import types
import warnings

import numpy as np
import pytest
from scipy.special import ndtr

import grad_oracle as GO
import logei_oracle as LO
import mes_oracle as MO
from oracle import dd
from oracle import gp_oracle as O
from oracle import make_acq_big as AB
from oracle import make_illcond as MI
from test_gpu_illcond import RTOL, _order_keys
from test_gpu_illcond_big import PRUNE_SETTINGS
from test_gpu_illcond_ext import _grad_err, _order_ok
from test_gpu_logei import _key_value
from test_gpu_mes import _ENV, VARIANTS

pytestmark = pytest.mark.gpu

PROBLEMS = AB.PROBLEMS
SMALL_ROWS = 256  # the small-batch path runs on the first rows only
C_REF = 100.0
FLOOR = dict(log=1e-12, rel=1e-10, grad=1e-10)
# Bars at about 10x the measurement (comments) per problem and family of kinds, over the fp64 variants and the
# incumbent levels: "log" LogEI / LogPoI, "mes" MES, "base" UCB / EI / PoI, "prod" EI / PoI / MES x PoF, "logc" LogEI /
# LogPoI + sum log p.  A family the table does not name is held by the rule alone.
PIN = {
    ("b_m05_ard", "log"): 1e-8,  # 9.8e-10
    ("b_m05_ard", "mes"): 2.2e-9,  # 2.2e-10
    ("b_m15_d17", "log"): 1.1e-6,  # 1.1e-7
    ("b_m15_d17", "mes"): 1e-8,  # 1.0e-9
    ("b_m15_d17", "prod"): 2.2e-8,  # 2.2e-9
    ("b_m15_d17", "logc"): 1.5e-3,  # 1.5e-4 (sigma of the RBF constraint GP at cond(K) 1.7e11)
    ("b_m25_c3", "log"): 4e-6,  # 4.0e-7
    ("b_m25_c3", "mes"): 1.3e-7,  # 1.3e-8
    ("b_m25_c3", "prod"): 6.4e-8,  # 6.4e-9
    ("b_m25_c3", "logc"): 1.1e-3,  # 1.1e-4 (the same; the referee's error is 1.1e-4 too)
    ("b_m25_c5", "base"): 3.4e-10,  # 3.4e-11
    ("b_m25_c5", "log"): 4.6e-6,  # 4.6e-7
    ("b_m25_c5", "mes"): 2.4e-7,  # 2.4e-8
    ("b_rbf_long", "log"): 1.3e-4,  # 1.3e-5
    ("b_rbf_long", "mes"): 1.2e-6,  # 1.2e-7
}
PIN_GRAD = {
    ("b_m05_ard", "log"): 5e-8,  # 5.0e-9
    ("b_m05_ard", "mes"): 2.5e-8,  # 2.5e-9
    ("b_m15_d17", "log"): 1.7e-6,  # 1.7e-7
    ("b_m15_d17", "mes"): 1.5e-6,  # 1.5e-7
    ("b_m15_d17", "prod"): 1.4e-10,  # 1.4e-11
    ("b_m15_d17", "logc"): 1.5e-3,  # 1.5e-4
    ("b_m25_c3", "log"): 9e-6,  # 9.0e-7
    ("b_m25_c3", "mes"): 5.1e-7,  # 5.1e-8
    ("b_m25_c3", "prod"): 6e-9,  # 6.0e-10
    ("b_m25_c3", "logc"): 2.2e-3,  # 2.2e-4
    ("b_m25_c5", "base"): 7.8e-8,  # 7.8e-9
    ("b_m25_c5", "log"): 6.9e-6,  # 6.9e-7
    ("b_m25_c5", "mes"): 2.2e-6,  # 2.2e-7
    ("b_rbf_long", "log"): 2.1e-4,  # 2.1e-5
    ("b_rbf_long", "mes"): 1e-10,  # 0 (every MES gradient row of the truth and the device is 0)
}
# fp32 mode, over the unconstrained kinds on the rows where sigma > 0.1 s_y (tests/test_gpu_illcond_big.py's rows),
# at 3x the measurement as BAR32_BIG pins b_m25_c3 there: past its stated bound at N in the thousands (DESIGN.md
# section 2) 10x would not bound anything.  The log kinds are measured on the rows where the fp32 value is finite: a
# non-finite one must sit on a row whose fp32 sigma^2 clamped to 0 (log 0 of the EI / PoI limit), and the number of
# such rows is pinned (FP32_CLAMPED).  b_rbf_long has no such rows.
BAR32 = {
    ("b_m05_ard", "log"): 3.6e-2,  # 1.2e-2
    ("b_m05_ard", "mes"): 3.9e-3,  # 1.3e-3
    ("b_m15_d17", "log"): 0.42,  # 1.4e-1
    ("b_m15_d17", "mes"): 9.3e-2,  # 3.1e-2
    ("b_m25_c3", "log"): 235.0,  # 78 (on the rows whose fp32 sigma^2 does not clamp)
    ("b_m25_c3", "mes"): 0.48,  # 1.6e-1
    ("b_m25_c5", "log"): 17.0,  # 5.6
    ("b_m25_c5", "mes"): 1.4,  # 4.6e-1
    ("b_m25_c5", "base"): 1.3,  # 4.2e-1
}
FP32_CLAMPED = {"b_m25_c3": 171}  # 57, at 3x
# Findings (DESIGN.md section 2), held to the pin instead of C_REF x the referee and the 1e-5 bar.  On b_rbf_long
# (cond(K) 1.8e11) LogEI and LogPoI carry sigma's residue c - sum V^2 of the product with the explicit inverse whole,
# as LogNEI does: 1.3e-5 against the referee's 5.9e-6 (values), 1.0e-5 against 2.9e-6 (gradients).  On b_m15_d17 the
# gradients of the log-space constrained forms miss 1e-5 (1.5e-4 against the referee's 8.2e-6, within C_REF): the
# RBF constraint GP's sigma, 9x further from the truth than the referee's at cond(K) 1.7e11, accounts for most of it
# (test_constrained_log_gradient_follows_the_device_sigma).
_LOG = [f"{k}_t{t}" for k in ("logei", "logpoi") for t in (0, 1, 4)]
FINDINGS = ({("b_rbf_long", k) for k in _LOG} | {("b_rbf_long", "g_" + k) for k in _LOG} |
            {("b_m15_d17", f"g_{k}_c_t{t}") for k in ("logei", "logpoi") for t in (0, 4)})
# (problem, key) where the lead stage's k-th value prunes every following tile of the eight-fold batch before the
# refine stage claims one (measured); in every other LogEI / LogPoI pair the refine stages evaluate candidates
# (measured 256 .. 32896 refined candidates).
NOT_REFINED = {("b_m05_ard", "logpoi_t0"), ("b_m15_d17", "logei_t0"), ("b_m15_d17", "logpoi_t0")}

_FIX, _GP = {}, {}
NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "rbf": np.inf}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = AB.load(name)
    return _FIX[name]


def _pin(monkeypatch, env):
    for k in _ENV + ("B200BO_PRUNE", "B200BO_PRUNE_REFINE", "B200BO_PRUNE_REFINE_BLOCKS", "B200BO_PRUNE_BOUND"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _gps(name):
    """(case, y) of the target and of each constraint GP."""
    r = fixture(name)
    out = [(AB.case(name), r["y"])]
    if name in AB.CONSTRAINED:
        out += list(zip(AB.constraint_cases(r["X"].shape[1]), (r["c0_y"], r["c1_y"])))
    return out


def _gp(bo, name, j=0, precision="fp64"):
    if (name, j, precision) not in _GP:
        c, y = _gps(name)[j]
        _GP[name, j, precision] = bo.B200GaussianProcessRegressor(
            kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True, optimizer=None,
            precision=precision).fit(fixture(name)["X"], y)
    return _GP[name, j, precision]


CODES = dict(ucb="ACQ_UCB", ei="ACQ_EI", poi="ACQ_POI", mes="ACQ_MES", logei="ACQ_LOGEI", logpoi="ACQ_LOGPOI")


def _acq(bo, name, key, precision="fp64", kappa=MI.KAPPA):
    from bayesianoptimization_b200 import _lib as B

    r = fixture(name)
    kind, p, form = AB.kinds(name)[key]
    cons = None
    if form is not None:
        b = [r["c0_bounds"], r["c1_bounds"]]
        cons = types.SimpleNamespace(model=[_gp(bo, name, 1, precision), _gp(bo, name, 2, precision)],
                                     lb=[v[0] for v in b], ub=[v[1] for v in b])
    extra = dict(max_values=r[f"ystar_{p}"]) if kind == "mes" else dict(y_max=float(r["y_max"][AB.T_LEVELS.index(p)]))
    return bo.FusedAcquisition(getattr(B, CODES[kind]), _gp(bo, name, 0, precision), constraint=cons, kappa=kappa,
                               xi=AB.XI, **extra)


def _is_log(key):
    return key.startswith("log")


def _family(key):
    if key in ("ucb", "ei", "poi"):
        return "base"
    if key.endswith("_pof"):
        return "prod"
    if "_c_t" in key:
        return "logc"
    return "mes" if key.startswith("mes") else "log"


def _value_err(key, got, want):
    with np.errstate(all="ignore"):
        if _is_log(key):
            e = np.abs(got - want) / (1.0 + np.abs(want))
        else:
            e = np.abs(got - want) / max(float(np.max(np.abs(want), initial=0.0)), np.finfo(float).tiny)
    return float(np.max(np.where(np.isfinite(e), e, np.inf), initial=0.0))


def _referee_values(name, key):
    """The referee's un-negated values of one kind at every candidate, from sklearn's mu and sigma."""
    r = fixture(name)
    kind, p, form = AB.kinds(name)[key]
    mu, sd = r["sk_mu"], r["sk_sd"]
    cons = [(r[f"sk_c{j}_mu"], r[f"sk_c{j}_sd"], *r[f"c{j}_bounds"]) for j in range(2)] if form else []
    with np.errstate(all="ignore"):
        if kind in ("logei", "logpoi"):
            code = LO.LOGEI if kind == "logei" else LO.LOGPOI
            return -LO.closure(code, mu, sd, float(r["y_max"][AB.T_LEVELS.index(p)]), AB.XI, cons)
        if kind == "mes":
            v = MO.mes_alpha(mu, sd, r[f"ystar_{p}"])
        else:
            code = {"ucb": O.ACQ_UCB, "ei": O.ACQ_EI, "poi": O.ACQ_POI}[kind]
            v = O.base_acq(code, mu, sd, kappa=MI.KAPPA, xi=AB.XI, y_max=float(r["y_max"][AB.T_LEVELS.index(p)]))
        for m, s, lb, ub in cons:
            v = v * (ndtr((ub - m) / s) - (0.0 if lb == -np.inf else ndtr((lb - m) / s)))
        return v


def _fmt(e):
    return " ".join(f"{k} {v:.1e}" for k, v in e.items())


def _hold(name, key, dev, ref, dev_all):
    """The rule on the rows where the referee forms a finite value (dev), the pin on every row (dev_all)."""
    if (name, key) not in FINDINGS:
        floor = FLOOR["log"] if _is_log(key) else FLOOR["rel"]
        assert dev <= max(C_REF * ref, floor), (name, key, dev, ref)
        if ref <= RTOL:
            assert dev <= RTOL, (name, key, dev, ref)
    pin = PIN.get((name, _family(key)))
    if pin is not None:
        assert dev_all <= pin, (name, key, dev_all)


# ---------------------------------------------------------------------------------------------------------------
# values through every variant; the constrained launches through the fp64 variants
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", PROBLEMS)
def test_values_against_truth(bo, monkeypatch, name, variant):
    r = fixture(name)
    fp32 = variant == "fp32"
    m = SMALL_ROWS if variant == "small" else len(r["xt"])
    _pin(monkeypatch, VARIANTS[variant])
    rows32 = r["sd"][:m] > 0.1 * float(np.std(r["y"]))
    worst, clamped32 = {}, 0
    if fp32:
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sd32 = _gp(bo, name, 0, "fp32").predict(r["xt"][:m], return_std=True)[1]
    for key, (kind, p, form) in AB.kinds(name).items():
        if fp32 and form is not None:
            continue
        got = -_acq(bo, name, key, "fp32" if fp32 else "fp64")(r["xt"][:m])
        want, sk = r[key][:m], _referee_values(name, key)[:m]
        if fp32:
            bad = rows32 & ~np.isfinite(got)
            # a non-finite value only where the fp32 sigma^2 clamped to 0: LogEI / LogPoI of the limit, log 0
            assert not bad.any() or (_is_log(key) and np.all(sd32[bad] == 0.0)), (key, np.flatnonzero(bad)[:5])
            clamped32 = max(clamped32, int(bad.sum()))
            fin = rows32 & np.isfinite(got)
            e = _value_err(key, got[fin], want[fin])
            print(f"\n{name} fp32 {key}: device {e:.1e} on {fin.sum()} rows ({bad.sum()} non-finite, sigma^2 clamped)")
            worst[_family(key)] = max(worst.get(_family(key), 0.0), e)
            continue
        ok = np.isfinite(sk)
        dev_all, dev, ref = _value_err(key, got, want), _value_err(key, got[ok], want[ok]), _value_err(key, sk[ok],
                                                                                                      want[ok])
        print(f"\n{name} {variant} {key}: device {dev_all:.1e} | referee {ref:.1e} on {ok.sum()} rows")
        _hold(name, key, dev, ref, dev_all)
    if fp32:
        print(f"{name} fp32: {clamped32} rows with sigma > 0.1 s_y clamp to sigma^2 = 0; worst {worst}")
        assert clamped32 <= FP32_CLAMPED.get(name, 0), clamped32
        for fam, e in worst.items():
            if (name, fam) in BAR32:
                assert e <= BAR32[name, fam], (fam, e)


# ---------------------------------------------------------------------------------------------------------------
# selection: the truth's order; pruning bit-equal, bound keys below exact keys, the margin's headroom
# ---------------------------------------------------------------------------------------------------------------
def _records(f, x, k=10):
    i, v, t = f.argmin_topk(x, k)
    return i, np.float64(v).view(np.int64), list(t)


def _bound_and_exact(B, f, x):
    import torch

    m = x.shape[0]
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    acq_o, kmax = (torch.empty(m, dtype=torch.float64, device="cuda") for _ in range(2))
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, acq_o.data_ptr(), None, None, 0, None, 0,
                                  s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), kmax.data_ptr(),
                                         s.cuda_stream))
    s.synchronize()
    return acq_o.cpu().numpy(), key.cpu().numpy().view(np.uint64)


def _order_ok_log(got, ref, tol):
    """_order_ok on the log kinds' metric: two candidates may trade places when their true values are within
    tol (1 + |v|) of each other."""
    want = [int(np.argmin(ref))] + list(np.argsort(ref, kind="stable")[:len(got) - 1])
    for g, w in zip(got, want):
        if g != w:
            assert abs(ref[g] - ref[w]) <= tol * (1 + max(abs(ref[g]), abs(ref[w]))), (g, w, ref[g], ref[w])


@pytest.mark.parametrize("name", PROBLEMS)
def test_selection_against_truth_and_pruning(bo, monkeypatch, name):
    from bayesianoptimization_b200 import _lib as B

    r = fixture(name)
    x = r["xt"]
    x8 = np.tile(x, (8, 1))
    near = np.isin(r["group"], (MI.G_TRAIN, MI.G_DUP7))
    headroom = {}
    for key, (kind, p, form) in AB.kinds(name).items():
        _pin(monkeypatch, {"B200BO_SMALL_PATH": "0"})
        f = _acq(bo, name, key)
        ref = -r[key]
        rec = _records(f, x)
        tol = 2 * PIN.get((name, _family(key)), RTOL)
        (_order_ok_log if _is_log(key) else _order_ok)([int(rec[0])] + [int(t) for t in rec[2]], ref, tol)
        if kind in ("logei", "logpoi") and form is None:
            out, refined = [], []
            for prune, refine, blocks in PRUNE_SETTINGS:
                _pin(monkeypatch, {"B200BO_SMALL_PATH": "0", "B200BO_PRUNE": prune, "B200BO_PRUNE_REFINE": refine,
                                   "B200BO_PRUNE_REFINE_BLOCKS": blocks})
                out.append(_records(f, x8))
                if prune == "1":
                    ms, ref_n = (C.c_float * 6)(), C.c_int64()
                    B.check(B.lib().b200bo_last_prune_stage_ms(ms, C.byref(ref_n)))
                    refined.append(ref_n.value)
            for bound in ("auto", "f64", "f32"):
                _pin(monkeypatch, {"B200BO_SMALL_PATH": "0", "B200BO_PRUNE": "1", "B200BO_PRUNE_BOUND": bound})
                out.append(_records(f, x8))
            print(f"\n{name} {key}: refined {refined}")
            assert all(o == out[0] for o in out[1:]), (key, out)
            assert refined[0] == 0, refined
            if (name, key) not in NOT_REFINED:
                assert refined[1] > 0 and refined[2] > 0, (key, refined)
            for bound in ("f64", "f32"):
                _pin(monkeypatch, {"B200BO_SMALL_PATH": "0", "B200BO_PRUNE_BOUND": bound})
                exact, keys = _bound_and_exact(B, f, x)
                bad = keys > _order_keys(exact)
                assert not bad.any(), (key, bound, f"{bad.sum()} bound keys above the exact key")
                live = near & (keys != 0) & np.isfinite(exact)
                if live.any():
                    gap = (exact[live] - _key_value(keys[live])) / (1e-9 * np.abs(exact[live]) + 1e-9)
                    headroom[key, bound] = float(gap.min())
        else:  # MES and the constrained kinds are outside pruning's scope
            out = []
            for prune in ("0", "1"):
                _pin(monkeypatch, {"B200BO_SMALL_PATH": "0", "B200BO_PRUNE": prune})
                out.append(_records(f, x8))
            assert out[0] == out[1], (key, out)
    # DESIGN.md 4.12: the smallest (exact - bound) on the training rows and their 1e-7 neighbours, in units of the
    # log kinds' margin 1e-9 |v| + 1e-9
    print(f"\n{name} margin headroom: " + " ".join(f"{k}/{b} {v:.2e}" for (k, b), v in sorted(headroom.items())))
    assert all(v > 0 for v in headroom.values()), headroom


# ---------------------------------------------------------------------------------------------------------------
# gradients on the 64 rows; clamped variances
# ---------------------------------------------------------------------------------------------------------------
def _referee_gp(c, X, y):
    return GO.GradGP(X, y, NU[c["kern"]], dd.ls_vec(c), const=float(c.get("const") or 1.0),
                     noise=float(c.get("white") or 0.0), alpha=c["alpha"])


def _referee_grads(name, rows):
    """{key: (value, gradient)} of the closure (negated), through tests/grad_oracle.py's fp64 GPs."""
    r = fixture(name)
    X = r["X"]
    preds = [_referee_gp(c, X, y).predict_grad(rows) for c, y in _gps(name)]
    mean, sd, dmean, dsd = preds[0]
    out = {}
    for key, (kind, p, form) in AB.kinds(name).items():
        cons = [(preds[j + 1], *r[f"c{j}_bounds"]) for j in range(2)] if form else []
        y_max = float(r["y_max"][AB.T_LEVELS.index(p)]) if kind != "mes" else 0.0
        with np.errstate(all="ignore"):
            if kind in ("logei", "logpoi"):
                code = LO.LOGEI if kind == "logei" else LO.LOGPOI
                v, cm, cs = LO.log_acq_term_grad(code, mean - y_max - AB.XI, sd)
                g = cm[:, None] * dmean + cs[:, None] * dsd
                for (m, s, dm, ds), lb, ub in cons:
                    v = v + LO.log_cfactor(lb, ub, m, s)
                    ccm, ccs = LO.log_cfactor_grad(lb, ub, m, s)
                    g = g + ccm[:, None] * dm + ccs[:, None] * ds
                out[key] = (-v, -g)
            else:
                code = {"ucb": GO.UCB, "ei": GO.EI, "poi": GO.POI, "mes": GO.MES}[kind]
                v, g = GO.base_value_grad(code, mean, sd, dmean, dsd, kappa=MI.KAPPA, xi=AB.XI, y_max=y_max,
                                          ystar=r[f"ystar_{p}"] if kind == "mes" else None)
                for (m, s, dm, ds), lb, ub in cons:
                    pj, dp = GO.prob_value_grad(lb, ub, m, s, dm, ds)
                    g = g * pj[:, None] + v[:, None] * dp
                    v = v * pj
                out[key] = (-v, -g)
    return out


@pytest.mark.parametrize("name", PROBLEMS)
def test_gradient_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    gi = r["grad_rows"]
    rows = r["xt"][gi]
    ls = np.concatenate([dd.ls_vec(c) for c, _ in _gps(name)])
    ref = _referee_grads(name, rows)
    worst = {}
    for key in AB.kinds(name):
        f = _acq(bo, name, key)
        _pin(monkeypatch, {})
        val, grad = f.value_and_grad(rows)
        _pin(monkeypatch, {"B200BO_SMALL_PATH": "1"})
        small = f(rows)
        assert np.array_equal(val.view(np.int64), small.view(np.int64)), key
        tv, tg = -r[key][gi], -r[f"g_{key}"]
        sv, sg = ref[key]
        e_dev, e_ref = _grad_err(grad, tg, tv, ls), _grad_err(sg, tg, tv, ls)
        ok = np.isfinite(e_ref)
        dev_all = float(np.max(np.where(np.isfinite(e_dev), e_dev, np.inf)))
        dev, rf = float(np.max(e_dev[ok], initial=0.0)), float(np.max(e_ref[ok], initial=0.0))
        print(f"\n{name} grad {key}: device {dev_all:.1e} | referee {rf:.1e} on {ok.sum()} rows")
        if (name, "g_" + key) not in FINDINGS:
            assert dev <= max(C_REF * rf, FLOOR["grad"]), (key, dev, rf)
            if rf <= RTOL:
                assert dev <= RTOL, (key, dev, rf)
        worst[_family(key)] = max(worst.get(_family(key), 0.0), dev_all)
    print(f"GRAD {name} worst {worst}")
    for fam, e in worst.items():
        if (name, fam) in PIN_GRAD:
            assert e <= PIN_GRAD[name, fam], (fam, e)


def _log_chain(r, name, key, sds):
    """The gradient of a log-space constrained closure (negated) on the grad rows, in fp64 from the truth's mu, d mu
    and d sigma^2 of each GP (gp<j>_*_g) with sigma = sds[j]: d sigma = d sigma^2 / (2 sigma)."""
    kind, p, _ = AB.kinds(name)[key]
    code = LO.LOGEI if kind == "logei" else LO.LOGPOI
    g = 0.0
    for j, sd in enumerate(sds):
        mu, dmu = r[f"gp{j}_mu_g"], r[f"gp{j}_dmu_g"]
        dsd = r[f"gp{j}_dsd_g"] * (r[f"gp{j}_sd_g"] / sd)[:, None]
        with np.errstate(all="ignore"):
            if j == 0:
                _, cm, cs = LO.log_acq_term_grad(code, mu - float(r["y_max"][AB.T_LEVELS.index(p)]) - AB.XI, sd)
            else:
                cm, cs = LO.log_cfactor_grad(*r[f"c{j - 1}_bounds"], mu, sd)
        g = g + cm[:, None] * dmu + cs[:, None] * dsd
    return -g


@pytest.mark.parametrize("name", AB.CONSTRAINED)
def test_constrained_log_gradient_follows_the_device_sigma(bo, monkeypatch, name):
    """The log-space constrained gradients on b_m15_d17 miss 1e-5 where the referee meets it (FINDINGS).  The truth's
    own chain rule, fed the device's sigma of each GP on the grad rows in place of the truth's (and so d sigma =
    d sigma^2 / (2 sigma_device)), is at least half as far from the truth as the device's gradient wherever that
    misses 1e-5: the device's sigma alone accounts for most of the error.  Measured on an H100 80GB HBM3 at 700 W:
    b_m15_d17 1.5e-4 against the device's 1.5e-4 (the device 6.6e-5 from that), b_m25_c3 1.4e-4 against 2.2e-4; the
    RBF constraint GP's sigma is 7.5e-5 from the truth on b_m15_d17 against the referee's 8.1e-6 (the residue
    c - sum V^2 of the product with the explicit inverse at cond(K) 1.7e11), 6.4e-5 against 5.6e-5 on b_m25_c3.  Prints
    the device's and the referee's sigma errors of each GP at every candidate."""
    r = fixture(name)
    gi = r["grad_rows"]
    rows = r["xt"][gi]
    ls = np.concatenate([dd.ls_vec(c) for c, _ in _gps(name)])
    for j in range(3):
        truth, sk = (r["sd"], r["sk_sd"]) if j == 0 else (r[f"c{j - 1}_sd"], r[f"sk_c{j - 1}_sd"])
        _pin(monkeypatch, {"B200BO_SMALL_PATH": "0"})
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            sd = _gp(bo, name, j).predict(r["xt"], return_std=True)[1]
        print(f"\n{name} gp{j} sigma: device {np.max(np.abs(sd - truth) / truth):.1e} | referee "
              f"{np.max(np.abs(sk - truth) / truth):.1e}")
    _pin(monkeypatch, {"B200BO_SMALL_PATH": "1"})
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sds = [_gp(bo, name, j).predict(rows, return_std=True)[1] for j in range(3)]
    _pin(monkeypatch, {})
    for key in (k for k in AB.kinds(name) if "_c_t" in k):
        tv, tg = -r[key][gi], -r[f"g_{key}"]
        grad = _acq(bo, name, key).value_and_grad(rows)[1]
        e_dev = float(np.max(_grad_err(grad, tg, tv, ls)))
        e_chain = float(np.max(_grad_err(_log_chain(r, name, key, [r[f"gp{j}_sd_g"] for j in range(3)]), tg, tv, ls)))
        g_sub = _log_chain(r, name, key, sds)
        e_sub = float(np.max(_grad_err(g_sub, tg, tv, ls)))
        e_res = float(np.max(_grad_err(grad, g_sub, tv, ls)))
        print(f"{name} {key}: device {e_dev:.1e}; truth with the device's sigma {e_sub:.1e}, device against that "
              f"{e_res:.1e}; fp64 chain on the rounded truth {e_chain:.1e}")
        assert e_chain <= 1e-2 * max(e_dev, FLOOR["grad"]), (key, e_chain, e_dev)
        if e_dev > RTOL:
            assert e_sub >= 0.5 * e_dev, (key, e_sub, e_dev)


@pytest.mark.parametrize("name", PROBLEMS)
def test_clamped_rows_follow_the_limit_rules(bo, monkeypatch, name):
    """Wherever the device clamps sigma^2 to 0 on the 64 gradient rows (the small-batch path, whose sigma the
    gradient's value shares bit for bit), DESIGN.md 4.10 / 4.12: d sd = 0 (UCB's gradient is the mean's), the PoI and
    MES coefficients are 0, LogEI and LogPoI take the log of their limit.  Prints how many rows clamped."""
    r = fixture(name)
    rows = r["xt"][r["grad_rows"]]
    gp = _gp(bo, name)
    _pin(monkeypatch, {"B200BO_SMALL_PATH": "1"})
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        mu, sd = gp.predict(rows, return_std=True)
    clamped = sd == 0.0
    print(f"\n{name}: {int(clamped.sum())} clamped rows of {len(rows)}")
    assert clamped.any() == any("smaller than 0" in str(x.message) for x in w)
    if not clamped.any():
        return
    c = rows[clamped]
    y_max = float(r["y_max"][0])
    a = mu[clamped] - y_max - AB.XI
    _pin(monkeypatch, {})
    ucb = {k: _acq(bo, name, "ucb", kappa=k).value_and_grad(c)[1] if "ucb" in AB.kinds(name) else None
           for k in (0.0, MI.KAPPA)}
    if ucb[0.0] is not None:
        assert np.array_equal(ucb[0.0], ucb[MI.KAPPA])
    for key, (kind, p, form) in AB.kinds(name).items():
        if form is not None or p not in (0, "k4"):
            continue
        val, grad = _acq(bo, name, key).value_and_grad(c)
        if kind in ("poi", "mes"):
            assert np.all(grad == 0.0), key
        if kind == "mes":
            assert np.all(val == 0.0), key
        with np.errstate(divide="ignore"):
            if kind == "logei":
                np.testing.assert_array_equal(val, -np.log(np.maximum(a, 0.0)))
            if kind == "logpoi":
                np.testing.assert_array_equal(val, -np.log((a > 0).astype(float)))

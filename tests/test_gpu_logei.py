"""LogEI and LogPoI on the H100: the log-space epilogue of the fused predict kernel against the numpy restatement
(tests/logei_oracle.py) evaluated on the device's own mu and sigma, through every predict kernel variant and every
predict case of tests/kernel_matrix_cases.py, with two constraint GPs in one launch; exp(LogEI) against the device's
EI; selection records; pruning on and off and the bound keys; value_and_grad against central differences of the
oracle and its independence of the batch position; KrigingBeliever batches; and the late-stage refinement that
motivates the feature.

Every case prints its measured error (pytest -s).  A late-stage incumbent (y_max = max y + s_y) puts most candidates
many sigma below it, where EI underflows."""
import ctypes as C
import warnings
from types import SimpleNamespace

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

import kernel_matrix_cases as KM
import logei_oracle as LO

pytestmark = pytest.mark.gpu

ALPHA, XI = 1e-6, 0.01
VARIANTS = {  # environment of each kernel variant (read per launch), as in tests/test_gpu_mes.py
    "m16n8k4": {"B200BO_SMALL_PATH": "0"},
    "pipe_cpasync": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_PIPE": "cpasync"},
    "pipe_bulk_mc": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_PIPE": "bulk"},
    "m8n8k4": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_MMA": "884"},
    "warps8": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_WARPS": "8"},
    "dfma": {"B200BO_SMALL_PATH": "0", "B200BO_PREDICT_IMPL": "dfma"},
    "small": {"B200BO_SMALL_PATH": "1"},
    "fp32": {"B200BO_SMALL_PATH": "0"},
}
_ENV = ("B200BO_SMALL_PATH", "B200BO_PREDICT_MMA", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_IMPL", "B200BO_PREDICT_PIPE",
        "B200BO_PRUNE")

# Bars (metric |d| / (1 + |value|)), pinned at about 10x the error measured on an H100 80GB HBM3 (700 W power limit)
BAR_EPI = 2e-14          # device epilogue against the restatement on the device's own mu, sigma: measured 1.5e-15
BAR_CONS = 2e-14         # two constraint GPs, their mu, sigma from the GPs' own predict calls: measured 1.3e-15
BAR_GRAD = 1e-4          # value_and_grad against central differences of the oracle (step 1e-5 length scales):
                         # measured at most 1.3e-5 (p11), the differences' own truncation and round-off


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _pin(monkeypatch, variant):
    for k in _ENV:
        monkeypatch.delenv(k, raising=False)
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)


def _eval_dev(bo, f, xt):
    """One b200bo_acq_eval_dev call: (mu, sd, closure values) of the same launch."""
    import torch

    B = bo._lib
    x = torch.from_numpy(np.ascontiguousarray(xt)).cuda()
    m = x.shape[0]
    acq, mu, sd = (torch.empty(m, dtype=torch.float64, device="cuda") for _ in range(3))
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(f.spec), x.data_ptr(), m, acq.data_ptr(), mu.data_ptr(),
                                        sd.data_ptr(), 0, None, 0, None))
    torch.cuda.synchronize()
    return mu.cpu().numpy(), sd.cpu().numpy(), acq.cpu().numpy()


def _err(v, ref):
    """max |d| / (1 + |ref|) over finite rows; the non-finite pattern (inf sign, NaN) must agree."""
    fin = np.isfinite(ref)
    assert np.array_equal(np.isnan(v), np.isnan(ref)) and np.array_equal(v[~fin & ~np.isnan(ref)],
                                                                        ref[~fin & ~np.isnan(ref)])
    return float(np.max(np.abs(v[fin] - ref[fin]) / (1.0 + np.abs(ref[fin])))) if fin.any() else 0.0


def _candidates(c, X, d, rs):
    uni = KM.inputs(c, 2000, d, rs)
    train = X[rs.choice(len(X), 16, replace=False)]
    near = X[rs.choice(len(X), 16, replace=False)] + 1e-7 * rs.choice([-1.0, 1.0], size=(16, d))
    far = 1e4 * np.max(KM.length_scale(c, d)) * (1.0 + rs.uniform(size=(16, d)))
    return np.vstack([uni, train, near, far])


_CACHE = {}


def _case(bo, cid, prec="fp64"):
    if cid not in _CACHE:
        c = KM.PREDICT[cid]
        n, d = c["n"], c["d"]
        X, y, rs = KM.problem(c, n, d, 300 + sorted(KM.PREDICT).index(cid))
        _CACHE[cid] = SimpleNamespace(c=c, X=X, y=y, d=d, xt=_candidates(c, X, d, rs), gps={},
                                      y_max=float(np.max(y) + np.std(y)))
    r = _CACHE[cid]
    if prec not in r.gps:
        r.gps[prec] = bo.B200GaussianProcessRegressor(kernel=KM.kernel(r.c, r.d), alpha=ALPHA, normalize_y=True,
                                                      optimizer=None, precision=prec).fit(r.X, r.y)
    return r


def _check_order(idx, top, v, ref):
    """argmin / top-10 records against the oracle's order; where they differ the values must tie within BAR_EPI."""
    want = [int(np.argmin(ref))] + list(np.argsort(ref, kind="stable")[:len(top)])
    got = [int(idx)] + [int(t) for t in top]
    for g, w in zip(got, want):
        if g != w:
            assert abs(ref[g] - ref[w]) <= 10 * BAR_EPI * (1.0 + abs(ref[w])), (g, w, ref[g], ref[w])


# ---------------------------------------------------------------------------------------------------------------
# the epilogue on every variant and case
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_log_kinds_against_the_oracle(bo, monkeypatch, cid, variant):
    B = bo._lib
    r = _case(bo, cid, "fp32" if variant == "fp32" else "fp64")
    gp = r.gps["fp32" if variant == "fp32" else "fp64"]
    _pin(monkeypatch, variant)
    fe = bo.FusedAcquisition(B.ACQ_EI, gp, xi=XI, y_max=r.y_max)
    mu, sd, ei_neg = _eval_dev(bo, fe, r.xt)
    ei = -ei_neg
    out, ei_err = [], 0.0
    for kind in (B.ACQ_LOGEI, B.ACQ_LOGPOI):
        f = bo.FusedAcquisition(kind, gp, xi=XI, y_max=r.y_max)
        mu2, sd2, v = _eval_dev(bo, f, r.xt)
        assert np.array_equal(mu2, mu) and np.array_equal(sd2, sd)  # the same phase A / B: only the epilogue differs
        ref = LO.closure(kind, mu, sd, r.y_max, XI)
        e = _err(v, ref)
        out.append(e)
        assert e <= BAR_EPI, (kind, e)
        idx, val, top = f.argmin_topk(r.xt, 10)
        assert val == v[idx] or (np.isnan(val) and np.isnan(v[idx]))
        _check_order(idx, top, v, ref)
        if kind == B.ACQ_LOGEI:
            # exp(LogEI) is the device's EI where that is representable, to EI's own round-off: phi(z) and Phi(z)
            # carry a relative error of about eps z^2 (from the exponent -z^2/2) and a Phi(z) + sigma phi(z) cancels
            # by another factor z^2 (measured up to 941 eps z^2, within 64 eps z^4)
            rows = ei > 1e-250
            z = (mu[rows] - r.y_max - XI) / sd[rows]
            rel = np.abs(np.exp(-v[rows]) - ei[rows]) / ei[rows]
            lim = 64 * np.finfo(float).eps * np.maximum(1.0, z * z) ** 2
            ei_err = max(ei_err, float(np.max(rel / (np.finfo(float).eps * np.maximum(1.0, z * z)))))
            assert np.all(rel <= lim), float(np.max(rel / lim))
            zero = (ei == 0.0) & (sd > 0.0)
            assert np.all(np.isfinite(v[zero]))  # finite where EI underflowed, and equal to the oracle (above)
            n_zero = int(zero.sum())
    print(f"{cid} {variant}: LogEI {out[0]:.1e}, LogPoI {out[1]:.1e}; exp(LogEI) vs EI {ei_err:.1f} eps z^2; "
          f"rows with EI = 0 and sigma > 0: {n_zero} of {len(r.xt)}")


def _constrained(bo, cid, n_cons=2):
    c = KM.CONSTRAINED[cid]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(KM.CONSTRAINED_TARGET, n, d, 400 + sorted(KM.CONSTRAINED).index(cid))
    s = X.sum(1) / np.sqrt(d)
    cv = np.column_stack([np.cos(2 * s), np.sin(3 * s) + 0.3 * X[:, 0]])[:, :n_cons]
    xt = _candidates(KM.CONSTRAINED_TARGET, X, d, rs)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(KM.CONSTRAINED_TARGET, d), alpha=ALPHA, normalize_y=True,
                                         optimizer=None).fit(X, y)
    lb = np.array([lo for _, lo, _ in KM.CONSTRAINTS[:n_cons]])
    ub = np.array([hi for _, _, hi in KM.CONSTRAINTS[:n_cons]])
    cm = bo.ConstraintModel(None, lb, ub)
    for m_, (spec, _, _) in zip(cm.model, KM.CONSTRAINTS[:n_cons]):
        m_.set_params(kernel=KM.kernel(spec, d), alpha=ALPHA, normalize_y=True, optimizer=None)
    cm.fit(X, cv)
    return SimpleNamespace(X=X, y=y, xt=xt, gp=gp, cm=cm, d=d, y_max=float(np.max(y) + np.std(y)), c=c)


@pytest.mark.parametrize("variant", [v for v in VARIANTS if v != "fp32"])
@pytest.mark.parametrize("cid", sorted(KM.CONSTRAINED))
def test_two_constraints_in_log_space(bo, monkeypatch, cid, variant):
    B = bo._lib
    r = _constrained(bo, cid)
    _pin(monkeypatch, variant)
    preds = [m_.predict(r.xt, return_std=True) for m_ in r.cm.model]
    cons = [(m_, s_, lo, hi) for (m_, s_), lo, hi in zip(preds, r.cm.lb, r.cm.ub)]
    errs = []
    for kind in (B.ACQ_LOGEI, B.ACQ_LOGPOI):
        f = bo.FusedAcquisition(kind, r.gp, r.cm, xi=XI, y_max=r.y_max)
        mu, sd, v = _eval_dev(bo, f, r.xt)
        ref = LO.closure(kind, mu, sd, r.y_max, XI, cons)
        errs.append(_err(v, ref))
        assert errs[-1] <= BAR_CONS
        idx, val, top = f.argmin_topk(r.xt, 10)
        assert val == v[idx] and idx == int(np.argmin(v))
    print(f"C {cid} {variant}: LogEI {errs[0]:.1e}, LogPoI {errs[1]:.1e}")


# ---------------------------------------------------------------------------------------------------------------
# pruning
# ---------------------------------------------------------------------------------------------------------------
def _order_keys(v):
    v = np.where(v == 0.0, 0.0, v)
    u = v.view(np.uint64)
    key = np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    return np.where(np.isnan(v), np.uint64(0xFFFFFFFFFFFFFFFF), key)


def _key_value(key):
    """Inverse of ordered_bits for keys of non-NaN values."""
    u = np.where(key >> np.uint64(63), key & ~np.uint64(1 << 63), ~key)
    return u.view(np.float64)


@pytest.mark.parametrize("kind", ["logei", "logpoi"])
@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_pruning_bit_equal_and_bound_below_exact(bo, monkeypatch, cid, kind):
    import torch

    B = bo._lib
    r = _case(bo, cid)
    _pin(monkeypatch, "m16n8k4")
    code = B.ACQ_LOGEI if kind == "logei" else B.ACQ_LOGPOI
    f = bo.FusedAcquisition(code, r.gps["fp64"], xi=XI, y_max=r.y_max)
    rs = np.random.RandomState(5)
    x = np.vstack([KM.inputs(r.c, 30_000, r.d, rs), r.xt])
    monkeypatch.setenv("B200BO_PRUNE", "0")
    off = f.argmin_topk(x, 10)
    monkeypatch.setenv("B200BO_PRUNE", "1")
    on = f.argmin_topk(x, 10)
    ev, tot = C.c_int64(), C.c_int64()
    B.check(B.lib().b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
    assert off[0] == on[0] and np.float64(off[1]).view(np.int64) == np.float64(on[1]).view(np.int64)
    assert list(off[2]) == list(on[2])
    # the device's bound keys against the keys of the exact values of the same candidates
    m = x.shape[0]
    xd = torch.from_numpy(x).cuda()
    acq_o, kmax = (torch.empty(m, dtype=torch.float64, device="cuda") for _ in range(2))
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, acq_o.data_ptr(), None, None, 0, None, 0,
                                  s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), kmax.data_ptr(),
                                         s.cuda_stream))
    s.synchronize()
    exact = acq_o.cpu().numpy()
    key = key.cpu().numpy().view(np.uint64)
    assert not np.any(key > _order_keys(exact))
    live = (key != 0) & np.isfinite(exact)
    gap = exact[live] - _key_value(key[live])  # how far below the exact value the bound sits, margin included
    print(f"{cid} {kind}: evaluated {ev.value} of {tot.value}; never-pruned {int((key == 0).sum())}; "
          f"min gap {gap.min():.2e}")


# ---------------------------------------------------------------------------------------------------------------
# gradients
# ---------------------------------------------------------------------------------------------------------------
def _oracle_closure(kind, gp, y_max, cm=None):
    def f(x):
        mu, sd = gp.predict(x, return_std=True)
        cons = []
        if cm is not None:
            cons = [(*m_.predict(x, return_std=True), lo, hi) for m_, lo, hi in zip(cm.model, cm.lb, cm.ub)]
        return LO.closure(kind, mu, sd, y_max, XI, cons)

    return f


def _fd_check(f_dev, f_or, xt, ls, d_float):
    val, grad = f_dev.value_and_grad(xt)
    fd = np.zeros_like(grad)
    for j in range(d_float):
        h = np.zeros(xt.shape[1])
        h[j] = 1e-5 * ls[j]
        fd[:, j] = (f_or(xt + h) - f_or(xt - h)) / (2 * h[j])
    g = grad[:, :d_float]
    scale = np.max(np.abs(fd[:, :d_float]), axis=1) + np.abs(val) / np.min(ls) + 1e-6
    return float(np.max(np.max(np.abs(g - fd[:, :d_float]), axis=1) / scale)), val, grad


@pytest.mark.parametrize("cid", sorted(KM.PREDICT))
def test_value_and_grad_against_central_differences(bo, monkeypatch, cid):
    B = bo._lib
    r = _case(bo, cid)
    _pin(monkeypatch, "small")
    rs = np.random.RandomState(8)
    uni = KM.inputs(r.c, 16, r.d, rs)
    near = r.X[rs.choice(len(r.X), 8, replace=False)] + 1e-3 * rs.choice([-1.0, 1.0], size=(8, r.d))
    xt = np.vstack([uni, near])
    ls = np.asarray(KM.length_scale(r.c, r.d), dtype=float) * np.ones(r.d)
    d_float = r.d - r.c.get("rnd", 0)
    out = []
    for kind in (B.ACQ_LOGEI, B.ACQ_LOGPOI):
        f = bo.FusedAcquisition(kind, r.gps["fp64"], xi=XI, y_max=r.y_max)
        e, val, grad = _fd_check(f, _oracle_closure(kind, r.gps["fp64"], r.y_max), xt, ls, d_float)
        assert np.array_equal(val, f(xt)) and np.all(np.isfinite(grad))
        if d_float < r.d:
            assert np.all(grad[:, d_float:] == 0.0)
        out.append(e)
        assert e <= BAR_GRAD
    print(f"grad {cid}: LogEI {out[0]:.1e}, LogPoI {out[1]:.1e}")


@pytest.mark.parametrize("cid", sorted(KM.CONSTRAINED))
def test_value_and_grad_two_constraints(bo, monkeypatch, cid):
    B = bo._lib
    r = _constrained(bo, cid)
    _pin(monkeypatch, "small")
    xt = r.xt[:24]
    ls = np.asarray(KM.length_scale(KM.CONSTRAINED_TARGET, r.d), dtype=float) * np.ones(r.d)
    for kind in (B.ACQ_LOGEI, B.ACQ_LOGPOI):
        f = bo.FusedAcquisition(kind, r.gp, r.cm, xi=XI, y_max=r.y_max)
        e, _, _ = _fd_check(f, _oracle_closure(kind, r.gp, r.y_max, r.cm), xt, ls, r.d)
        print(f"grad C {cid} kind {kind}: {e:.1e}")
        assert e <= BAR_GRAD


@pytest.mark.parametrize("cid", ["p2", "p5"])
def test_rows_do_not_depend_on_batch_position(bo, monkeypatch, cid):
    B = bo._lib
    r = _case(bo, cid)
    _pin(monkeypatch, "small")
    big = KM.inputs(r.c, 300, r.d, np.random.RandomState(9))
    for kind in (B.ACQ_LOGEI, B.ACQ_LOGPOI):
        f = bo.FusedAcquisition(kind, r.gps["fp64"], xi=XI, y_max=r.y_max)
        val, grad = f.value_and_grad(big)
        assert np.array_equal(val, f(big))
        row = big[7]
        v1, g1 = f.value_and_grad(row)
        assert v1[0] == val[7] and np.array_equal(g1[0], grad[7])
        for pos in (31, 32, 33, 299):
            batch = big.copy()
            batch[pos] = row
            v, g = f.value_and_grad(batch[:max(pos + 1, 34)] if pos < 299 else batch)
            assert v[pos] == val[7] and np.array_equal(g[pos], grad[7])


# ---------------------------------------------------------------------------------------------------------------
# through the acquisition classes
# ---------------------------------------------------------------------------------------------------------------
def test_kriging_believer_batch(bo, ref):
    opt = ref.BayesianOptimization(f=lambda x, y: -(x - 0.3) ** 2 - (y + 0.2) ** 2, pbounds={"x": (-1, 1), "y": (-1, 1)},
                                   acquisition_function=bo.KrigingBeliever(bo.LogExpectedImprovement(xi=0.01)),
                                   random_state=2, verbose=0)
    bo.enable(opt)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        opt.maximize(init_points=6, n_iter=2)
        pts = bo.suggest_batch(opt, 4)
    X = np.array([[p["x"], p["y"]] for p in pts])
    assert X.shape == (4, 2) and len({x.tobytes() for x in X}) == 4
    assert len(opt._acquisition_function.dummies) >= 4


def _late_stage(d, n, seed):
    """A late-stage training set: a fifth of the rows uniform, the rest clustered around the optimum with a spread
    shrinking from 1e-1 to 1e-3 (the study of DESIGN.md 4.12)."""
    rs = np.random.RandomState(seed)
    opt = np.full(d, 0.6)
    n_u = n // 5
    spread = np.logspace(-1, -3, n - n_u)[:, None]
    X = np.vstack([rs.uniform(size=(n_u, d)), np.clip(opt + spread * rs.randn(n - n_u, d), 0.0, 1.0)])
    y = -np.sum((X - opt) ** 2, axis=1)
    return X, y


def test_late_stage_refinement_moves_where_ei_cannot(bo, ref, monkeypatch):
    """d = 2, N = 60: EI's refinement runs from its top seeds take no iteration (EI is about 1e-9 at its best and its
    gradient is below gtol); LogEI's move, and its suggestion is no worse in LogEI than EI's."""
    from bayesianoptimization_b200 import acquisition as A

    d = 2
    X, y = _late_stage(d, 60, 1)
    opt = ref.BayesianOptimization(f=None, pbounds={f"x{j:02d}": (0.0, 1.0) for j in range(d)}, random_state=1,
                                   verbose=0, acquisition_function=bo.LogExpectedImprovement(xi=0.01))
    for x, t in zip(X, y):
        opt.register(opt.space.array_to_params(x), float(t))
    bo.enable(opt)
    opt.set_gp_params(kernel=Matern(nu=2.5, length_scale=1.0, length_scale_bounds="fixed"), optimizer=None,
                      alpha=1e-6, normalize_y=True)
    runs = {}
    real = A.lockstep_lbfgsb

    def recording(acq, seeds, bounds, *a, **kw):
        out = real(acq, seeds, bounds, *a, **kw)
        runs.setdefault(acq.kind, []).append([(int(o.nit), float(np.linalg.norm(o.x - s))) for o, s in zip(out, seeds)])
        return out

    monkeypatch.setattr(A, "lockstep_lbfgsb", recording)
    picks = {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for acq in (bo.ExpectedImprovement(xi=0.01), bo.LogExpectedImprovement(xi=0.01)):
            picks[type(acq).__name__] = acq.suggest(opt._gp, opt.space, n_random=10_000, n_smart=5,
                                                    random_state=np.random.RandomState(7))
    ei_runs, log_runs = runs[bo._lib.ACQ_EI][0], runs[bo._lib.ACQ_LOGEI][0]
    print(f"late stage: EI runs (nit, moved) {ei_runs}; LogEI runs {log_runs}")
    assert all(nit == 0 for nit, _ in ei_runs)
    assert any(nit > 0 for nit, _ in log_runs)
    le = bo.LogExpectedImprovement(xi=0.01)
    le.y_max = float(np.max(y))
    f = bo.FusedAcquisition(bo._lib.ACQ_LOGEI, opt._gp, owner=le)
    v = f(np.vstack([picks["LogExpectedImprovement"], picks["ExpectedImprovement"]]))
    print(f"late stage: -LogEI at LogEI's pick {v[0]:.6g}, at EI's pick {v[1]:.6g}")
    assert v[0] <= v[1]

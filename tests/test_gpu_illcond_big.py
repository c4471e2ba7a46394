"""The fit, posterior, pruned selection and Kriging-believer conditioning at production sizes on ill-conditioned
training sets, against a double-double reference.

tests/test_gpu_illcond.py and tests/test_gpu_illcond_ext.py referee the device on clustered, ill-conditioned sets
against 50 digits, but only up to N = 200.  The fixtures here (oracle/make_illcond_big.py, tests/golden/illbig_*.npz)
reach N = 1000 .. 4096 with cond(K) from 1e7 to 1e11 and hold the double-double truth (oracle/dd.py) and sklearn's fp64
results on the same rows.  At these sizes the look-ahead Cholesky runs over up to 64 diagonal steps, the explicit
inverse L^-1 over up to 64 blocks, phase B of the predict kernel over up to 32 row blocks, the refine stages of pruning
run (N > 896, at least 32 candidate tiles), and conditioning b_m25_c3 (np = N = 4096) re-pitches every N^2 buffer at the
first pending row.

The rules are those of tests/test_gpu_illcond.py (its C_SK and FLOOR): device error <= max(C_SK * sklearn's error,
FLOOR), the 1e-5 bar wherever sklearn meets it, and per-case bars pinned at about 10x the error measured on an H100
80GB HBM3 at a 700 W power limit (in the comments).  Every case prints the device's and sklearn's errors (pytest -s).
"""
import ctypes as C
import warnings

import numpy as np
import pytest

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_illcond_big as MB
from test_gpu_illcond import (BAR32, C_SK, FIT_PATHS, FLOOR, RTOL, RTOL32, _e32, _errors, _fmt, _hold, _order_keys,
                              _sk_errors)
from test_gpu_illcond_ext import _chain, _order_ok
from test_gpu_mes import _ENV, VARIANTS

pytestmark = pytest.mark.gpu

CASES = sorted(MB.CASES)
SMALL_ROWS = 256  # the small-problem path runs on the first rows only

# Per-case bars, pinned at about 10x the measurement (comments): PREDICT_BAR over mu, sigma, UCB, EI, PoI and the
# seven fp64 variants; FIT_BAR over diag(L), the stored rows of L and alpha_ on the five factorisation paths, the LML
# and its gradient; RES_BAR on the residual of alpha_ (2x, as in tests/test_gpu_illcond.py: it is deterministic);
# COND_BAR over the conditioned pivots, believer targets, mu and sigma (both forms, every fp64 variant).
PREDICT_BAR = {
    "b_m05_ard": 2e-7,  # 2.0e-8
    "b_m15_d17": 8e-7,  # 7.9e-8
    "b_m25_c3": 2e-6,  # 2.0e-7
    "b_rbf_long": 5e-3,  # 4.9e-4 (UCB at cond 1.8e11; sklearn's own error is 7.5e-4)
}
FIT_BAR = {
    "b_m05_ard": 5e-11,  # 5.0e-12
    "b_m15_d17": 5.5e-8,  # 5.4e-9
    "b_m25_c3": 1.7e-7,  # 1.6e-8
    "b_rbf_long": 2.4e-6,  # 2.3e-7
}
RES_BAR = {  # the same on every path
    "b_m05_ard": 7.6e-15,  # 3.7e-15
    "b_m15_d17": 2.5e-13,  # 1.2e-13
    "b_m25_c3": 8.4e-13,  # 4.1e-13
    "b_rbf_long": 2.7e-7,  # 1.3e-7
}
COND_BAR = {
    "b_m05_ard": 5e-9,  # 4.9e-10
    "b_m15_d17": 6.1e-7,  # 6.1e-8
    "b_m25_c3": 1.7e-6,  # 1.6e-7
    "b_rbf_long": 1.5e-4,  # 1.4e-5
}
# fp32 mode, DESIGN.md section 2.  Its stated bound |d sigma^2| <= 1e-3 sigma^2 + 1e-4 prior s_y^2 (BAR32) holds on
# b_m05_ard and b_rbf_long but not at cond(K) ~ 1e9 and N in the thousands: the 3xTF32 products of phase B accumulate
# in fp32 over N terms, and sigma^2 = prior - sum V^2 is a small residue of terms of order |L^-1| |k*|.  Those cases are
# pinned at their measurement instead (b_m25_c3 at 3x: 10x would not bound anything).  ACQ32: the acquisitions where
# sigma > 0.1 s_y, max |a - a_true| / (|a_true| + max |a_true|), below RTOL32 (tests/test_gpu_illcond.py's rule).
BAR32_BIG = {
    "b_m15_d17": 5e-2,  # 4.7e-3
    "b_m25_c3": 0.35,  # 1.1e-1
}
ACQ32_BIG = {
    "b_m05_ard": 2.1e-2,  # 2.1e-3
    "b_m15_d17": 0.23,  # 2.3e-2
    "b_m25_c3": 0.9,  # 3.0e-1 (3x)
}
# (case, kind) where the refine stages evaluate candidates of the eight-fold batch, with the measured count of refined
# candidates (one leading row block); in the other pairs the lead stage's k-th value prunes every following tile before
# the refine stage claims one.  The counts depend on the order in which the SMs claim tiles (b_rbf_long measured 16896
# to 17664 over two runs); the records do not.
REFINED = {("b_m05_ard", "ucb"): 4864, ("b_m05_ard", "ei"): 256, ("b_m15_d17", "ucb"): 512,
           ("b_m25_c3", "ucb"): 3712, ("b_m25_c3", "ei"): 2432, ("b_m25_c3", "poi"): 1280,
           ("b_rbf_long", "ei"): 16896, ("b_rbf_long", "poi"): 16896}

_FIX = {}


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def fixture(name):
    if name not in _FIX:
        _FIX[name] = MB.load(name)
    return _FIX[name]


def _rows(r, m):
    """The fixture restricted to its first m candidates."""
    return {k: v[:m] if isinstance(v, np.ndarray) and v.shape[:1] == r["mu"].shape else v for k, v in r.items()}


def _quiet(fn, *a, **k):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return fn(*a, **k)


def _pin(monkeypatch, variant):
    for k in _ENV + ("B200BO_PRUNE", "B200BO_PRUNE_REFINE", "B200BO_PRUNE_REFINE_BLOCKS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in VARIANTS[variant].items():
        monkeypatch.setenv(k, v)


def _gp(bo, name, precision="fp64"):
    c, r = MB.CASES[name], fixture(name)
    return bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"], normalize_y=True,
                                           optimizer=None, precision=precision).fit(r["X"], r["y"])


def _acq(bo, gp, kind, r):
    from bayesianoptimization_b200 import _lib as B

    code = {"ucb": B.ACQ_UCB, "ei": B.ACQ_EI, "poi": B.ACQ_POI}[kind]
    return bo.FusedAcquisition(code, gp, kappa=MI.KAPPA, xi=MI.XI, y_max=float(np.max(r["y"])))


# ---------------------------------------------------------------------------------------------------------------
# predict + acquisition through every kernel variant
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", CASES)
def test_predict_and_acquisition_against_truth(bo, monkeypatch, name, variant):
    r = fixture(name)
    if variant == "small":
        r = _rows(r, SMALL_ROWS)
    fp32 = variant == "fp32"
    gp = _gp(bo, name, "fp32" if fp32 else "fp64")
    _pin(monkeypatch, variant)
    xt = r["xt"]
    mu, sd = _quiet(gp.predict, xt, return_std=True)
    acq = {k: -_acq(bo, gp, k, r)(xt) for k in ("ucb", "ei", "poi")}
    dev, sk = _errors(r, mu, sd, acq), _sk_errors(r)
    print(f"\n{name} {variant} cond {float(r['cond']):.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    if fp32:
        e32 = _e32(r, sd, r["var"])
        rows = r["sd"] > 0.1 * r["y_std"]
        a32 = 0.0
        for k in ("ucb", "ei", "poi"):
            ref = r[f"acq_{k}"][rows]
            scale = max(float(np.max(np.abs(r[f"acq_{k}"]))), 1e-12)
            a32 = max(a32, float(np.max(np.abs(acq[k][rows] - ref) / (np.abs(ref) + scale), initial=0.0)))
        print(f"  fp32 e32 {e32:.1e} acq32 {a32:.1e} on {rows.sum()} rows")
        _hold(dev, sk, ("mu",))
        assert e32 <= BAR32_BIG.get(name, BAR32)
        assert a32 <= ACQ32_BIG.get(name, RTOL32)
        return
    _hold(dev, sk, ("mu", "sd", "ucb", "ei", "poi"))
    if name in PREDICT_BAR:
        assert max(dev.values()) <= PREDICT_BAR[name]


# ---------------------------------------------------------------------------------------------------------------
# selection: truth's order; pruning with and without the refine stages bit-equal; bound keys below the exact keys
# ---------------------------------------------------------------------------------------------------------------
PRUNE_SETTINGS = (("0", "1", "4"), ("1", "0", "4"), ("1", "1", "1"), ("1", "1", "4"))  # PRUNE, REFINE, REFINE_BLOCKS


@pytest.mark.parametrize("kind", ("ucb", "ei", "poi"))
@pytest.mark.parametrize("name", CASES)
def test_selection_against_truth_and_pruning(bo, monkeypatch, name, kind):
    import torch

    from bayesianoptimization_b200 import _lib as B

    r = fixture(name)
    gp = _gp(bo, name)
    f = _acq(bo, gp, kind, r)
    _pin(monkeypatch, "m16n8k4")
    x = r["xt"]
    ref = -r[f"acq_{kind}"]
    idx, val, top = f.argmin_topk(x, 10)
    _order_ok([int(idx)] + [int(t) for t in top], ref, 2 * PREDICT_BAR.get(name, RTOL))
    # Pruning on eight copies of the candidates (272 tiles): on the 34 tiles of the candidates alone the lead stage's
    # k-th value prunes every following tile in all but two of the twelve (case, kind) pairs; the copies give the
    # refine stage candidates to evaluate in eight of them, at least one kind per case (REFINED).
    x = np.tile(x, (8, 1))
    out, refined = [], []
    for prune, refine, blocks in PRUNE_SETTINGS:
        monkeypatch.setenv("B200BO_PRUNE", prune)
        monkeypatch.setenv("B200BO_PRUNE_REFINE", refine)
        monkeypatch.setenv("B200BO_PRUNE_REFINE_BLOCKS", blocks)
        i, v, t = f.argmin_topk(x, 10)
        out.append((i, np.float64(v).view(np.int64), list(t)))
        if prune == "1":
            ms, ref_n = (C.c_float * 6)(), C.c_int64()
            B.check(B.lib().b200bo_last_prune_stage_ms(ms, C.byref(ref_n)))
            refined.append(ref_n.value)
    print(f"\n{name} {kind}: refined {refined}")
    assert all(o == out[0] for o in out[1:]), out
    assert refined[0] == 0, refined  # B200BO_PRUNE_REFINE=0 keeps to the tile kernel
    if (name, kind) in REFINED:  # the refine stages looked at candidates with one and with four leading row blocks
        assert refined[1] > 0 and refined[2] > 0, refined
    m = x.shape[0]
    xd = torch.from_numpy(x).cuda()
    acq_o = torch.empty(m, dtype=torch.float64, device="cuda")
    key = torch.empty(m, dtype=torch.int64, device="cuda")
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, acq_o.data_ptr(), None, None, 0, None, 0,
                                  s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), None, s.cuda_stream))
    s.synchronize()
    bad = key.cpu().numpy().view(np.uint64) > _order_keys(acq_o.cpu().numpy())
    assert not bad.any(), f"{bad.sum()} bound keys above the exact key, e.g. row {np.flatnonzero(bad)[0]}"


# ---------------------------------------------------------------------------------------------------------------
# fit side: K, diag(L), rows of L, alpha_ and its residual through every factorisation path; LML and gradient
# ---------------------------------------------------------------------------------------------------------------
_DD = {}


def _dd_fit(name):
    if name not in _DD:
        r = fixture(name)
        _DD[name] = dd.Fit(MB.CASES[name], r["X"], r["y"])
    return _DD[name]


def _sk_K(name):
    c, r = MB.CASES[name], fixture(name)
    K = MI.sk_kernel(c)(r["X"])
    K[np.diag_indices_from(K)] += c["alpha"]
    return K


def _fit_errors(r, diag, rows, a):
    return dict(L=float(max(np.max(np.abs(diag - r["L_diag"]) / r["L_diag"]),
                            np.max(np.abs(rows - r["L_rows"])) / np.max(np.abs(r["L_rows"])))),
                alpha=float(np.max(np.abs(a - r["alpha_"])) / np.max(np.abs(r["alpha_"]))))


@pytest.mark.parametrize("path", list(FIT_PATHS))
@pytest.mark.parametrize("name", CASES)
def test_fit_state_against_truth(bo, monkeypatch, name, path):
    from bayesianoptimization_b200 import _lib as B

    for k in ("B200BO_POTRF", "B200BO_GEMM", "B200BO_GRAPH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in FIT_PATHS[path].items():
        monkeypatch.setenv(k, v)
    r = fixture(name)
    n = len(r["X"])
    gp = _gp(bo, name)
    K = np.empty((n, n))
    B.check(B.lib().b200bo_gp_get(gp._handle().ptr, B.GET_K, B.as_dp(K), n * n))
    ref = _dd_fit(name)
    Kt = ref.K[0] + ref.K[1]
    e_K = float(np.max(np.abs(K - Kt) / np.abs(Kt)))
    Ld = gp.L_
    idx = r["L_rows_idx"]
    dev = _fit_errors(r, np.diag(Ld), Ld[idx], gp.alpha_)
    sk = _fit_errors(r, r["sk_L_diag"], r["sk_L_rows"], r["sk_alpha_"])
    dev["res"] = ref.residual(K, gp.alpha_)
    sk["res"] = ref.residual(_sk_K(name), r["sk_alpha_"])
    print(f"\n{name} {path} cond {float(r['cond']):.1e}: K {e_K:.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    assert e_K <= 4e-16 * (1 + 2 * np.sqrt(MB.CASES[name]["d"]))
    _hold(dev, sk, ("L", "alpha", "res"))
    if name in FIT_BAR:
        assert max(dev["L"], dev["alpha"]) <= FIT_BAR[name]
    if name in RES_BAR:
        assert dev["res"] <= RES_BAR[name]


@pytest.mark.parametrize("name", CASES)
def test_lml_and_gradient_against_truth(bo, name):
    r = fixture(name)
    gp = _gp(bo, name)
    theta = MI.sk_kernel(MB.CASES[name]).theta
    lml, grad = gp.log_marginal_likelihood(theta, eval_gradient=True)
    gs = max(float(np.max(np.abs(r["lml_grad"]))), 1.0)
    dev = dict(lml=abs(lml - r["lml"]) / abs(r["lml"]), grad=float(np.max(np.abs(grad - r["lml_grad"]))) / gs)
    sk = dict(lml=abs(r["sk_lml"] - r["lml"]) / abs(r["lml"]),
              grad=float(np.max(np.abs(r["sk_lml_grad"] - r["lml_grad"]))) / gs)
    print(f"\n{name} lml cond {float(r['cond']):.1e}\n  device  {_fmt(dev)}\n  sklearn {_fmt(sk)}")
    assert grad.shape == r["lml_grad"].shape
    _hold(dev, sk, ("lml", "grad"))
    if name in FIT_BAR:
        assert max(dev.values()) <= FIT_BAR[name]


# ---------------------------------------------------------------------------------------------------------------
# Kriging-believer conditioning: 1, 8 and 64 pending rows, in one call and chained
# ---------------------------------------------------------------------------------------------------------------
def _cond_errors(r, p, mu, sd, tgt=None, piv=None):
    tsd = np.sqrt(r[f"inc_p{p}_var"])
    e = dict(mu=float(np.max(np.abs(mu - r["mu"]) / (np.abs(r["mu"]) + r["y_std"]))),
             sd=float(np.max(np.abs(sd - tsd) / tsd)))
    if tgt is not None:
        want = r["inc_target"][:p]
        e["target"] = float(np.max(np.abs(tgt - want) / (np.abs(want) + r["y_std"])))
        e["pivot"] = float(np.max(np.abs(piv - r["inc_pivot"][:p]) / r["inc_pivot"][:p]))
    return e


C_COND = dict(C_SK, target=30.0, pivot=100.0)  # tests/test_gpu_illcond_ext.py's C_REF on these metrics
FLOOR_COND = dict(FLOOR, target=1e-13, pivot=1e-11)


def _hold_cond(dev, ref):
    for k in dev:
        assert dev[k] <= max(C_COND[k] * ref[k], FLOOR_COND[k]), (k, dev[k], ref[k])
        if ref[k] <= RTOL:
            assert dev[k] <= RTOL, (k, dev[k], ref[k])


@pytest.mark.parametrize("name", CASES)
def test_conditioned_posterior_against_truth(bo, monkeypatch, name):
    r = fixture(name)
    gp = _gp(bo, name)
    n, xt, P = len(r["X"]), r["xt"], r["P"]
    worst = 0.0
    for p in MB.PREFIXES:
        ref = _cond_errors(r, p, r[f"sk_inc_p{p}_mu"], r[f"sk_inc_p{p}_sd"],
                           r["sk_inc_target"][:p], r["sk_inc_pivot"][:p])
        one = gp.condition_on_pending(P[:p])
        chained, forks, want = _chain(gp, P[:p])
        assert forks == want, (forks, want)
        for form, cg in (("one", one), ("chain", chained)):
            assert cg.X_train_.shape[0] == n + p
            fit = _cond_errors(r, p, r["mu"], np.sqrt(r[f"inc_p{p}_var"]), cg._y_raw[n:], np.diag(cg.L_)[n:])
            fit = {k: fit[k] for k in ("target", "pivot")}
            print(f"\n{name} p={p} {form} forks {forks}: {_fmt(fit)} | sklearn "
                  f"{_fmt({k: ref[k] for k in fit})}")
            _hold_cond(fit, {k: ref[k] for k in fit})
            worst = max(worst, *fit.values())
            for variant in VARIANTS:
                if variant in ("fp32", "small"):
                    continue
                _pin(monkeypatch, variant)
                mu, sd = _quiet(cg.predict, xt, return_std=True)
                dev = _cond_errors(r, p, mu, sd)
                print(f"  {variant:13s} device {_fmt(dev)} | sklearn {_fmt({k: ref[k] for k in dev})}")
                _hold_cond(dev, {k: ref[k] for k in dev})
                worst = max(worst, *dev.values())
    print(f"COND {name} worst {worst:.2e}")
    if name in COND_BAR:
        assert worst <= COND_BAR[name]

"""Selection-only pruning (DESIGN.md 4.9) across every prunable kind, a pairwise-covering set of its switches and
adversarial acquisition parameters, against the double-double truth of oracle/make_prune_matrix.py.

For every problem of tests/golden/prunemx_*.npz (d = 2, 5, 6, 16, 17, 32; N = 901 .. 4096, ragged against 64 and 128;
a 1e6 target offset with y_std 5e-4; ConstantKernel 2^-13 and 2^13 with a WhiteKernel term; cond(K) up to 1.8e11),
every kind (UCB, EI, PoI, LogEI, LogPoI) and every parameter point of the fixture (kappa -1, 0, 2.576, 100; y_max below
every mu, max y, max y + 4 s_y, each with xi 0, 0.01, 10 s_y):
  1. the records (argmin and top-k: value bits and indices) of every switch combination of SETTINGS (every pair of
     values of the four B200BO_PRUNE_* switches, and the defaults) equal those with B200BO_PRUNE=0, at k = 1 and
     k = 64 (B200BO_MAX_TOPK), on host candidates, on device candidates and on eight copies of the candidates (35 tiles,
     where the lead, refine, level and final stages run).  Each problem must have calls where the refine stage
     evaluated candidates and where the level let some through;
  2. the keys of the direct, fp64 Gram and fp32 Gram bound passes are never above the exact key of the device's value,
     and the Gram passes' mu interval holds the device's mu; the largest (max k*_i^2 / K_ii - sum V^2) / prior is
     reported against kPruneVarEps = 1e-8;
  3. the unpruned records are numpy's argmin and stable argsort of the device's own values (copies and PoI's exact 1.0
     resolve to the lowest index), and follow the truth's order up to swaps of values within twice the pin;
  4. check 1 (defaults and the single-switch arms) on a GP conditioned on pending rows that re-pitch np (a forked
     handle) and then conditioned again in place; on an fp32 handle pruning does not apply, and the records still
     equal those with B200BO_PRUNE=0.
Host rows with a NaN or +-inf coordinate are refused (ValueError) with pruning on and off; no candidate value here is
NaN (the NaN of sigma = 0 at a = 0 is never pruned: key 0, tests/test_prune_cpu.py).
"""
import ctypes as C
import itertools
import time

import numpy as np
import pytest

from oracle import make_illcond as MI
from oracle import make_prune_matrix as PM
from test_gpu_illcond import _order_keys
from test_prune_cpu import VAR_EPS

pytestmark = pytest.mark.gpu

SWITCHES = ("B200BO_PRUNE_REFINE", "B200BO_PRUNE_REFINE_BLOCKS", "B200BO_PRUNE_BOUND", "B200BO_PRUNE_GRAM_KERNEL")
VALUES = (("1", "0"), ("4", "1", "64"), ("auto", "f64", "f32"), ("reg", "ring"))
DEFAULTS = tuple(v[0] for v in VALUES)


def switch(setting, name):
    """the value of switch B200BO_PRUNE_<name> in a setting"""
    return setting[SWITCHES.index("B200BO_PRUNE_" + name)]


def pairwise(values):
    """A greedy covering array: every pair of values of every two switches appears in some row; the defaults first."""
    n = len(values)
    todo = {(i, a, j, b) for i, j in itertools.combinations(range(n), 2) for a in values[i] for b in values[j]}
    rows = [tuple(v[0] for v in values)]
    while True:
        todo -= {(i, r[i], j, r[j]) for r in rows[-1:] for i, j in itertools.combinations(range(n), 2)}
        if not todo:
            return rows
        rows.append(max(itertools.product(*values),
                        key=lambda r: sum((i, r[i], j, r[j]) in todo for i, j in itertools.combinations(range(n), 2))))


SETTINGS = pairwise(VALUES)
# the defaults and each switch's other values alone
SINGLE = [DEFAULTS] + [DEFAULTS[:i] + (v,) + DEFAULTS[i + 1:] for i, vs in enumerate(VALUES) for v in vs[1:]]
K_MAX = 64
# the pin of check 3 per problem: the largest device error against the truth (linear kinds: |d| / max |v|; log kinds:
# |d| / (1 + |v|)) over every kind and parameter point, about 10x the error measured on an H100 80GB HBM3 at a 700 W
# power limit and never below the floors of tests/test_gpu_acq_big.py (1e-10 linear, 1e-12 log).  On o_offset_d2
# a = mu - y_max - xi is a difference of two numbers near 1e6 whose fp64 rounding (1.2e-10) is large against sigma
# at the training copies (3e-8): the error is that of fp64 data units, not of the kernel.  Comments: measured linear, log.
PIN = {
    "b_m15_d17": (1.5e-8, 1.2e-6),  # 1.5e-9 1.2e-7
    "b_rbf_long": (3e-6, 1.2e-4),  # 2.9e-7 1.2e-5
    "b_m25_c3": (5e-8, 3e-6),  # 5.0e-9 2.9e-7
    "o_offset_d2": (5e-3, 8e-3),  # 5.0e-4 7.9e-4
    "o_clo_d5": (1e-10, 7.8e-12),  # 4.1e-12 7.8e-13
    "o_chi_d32": (8.6e-10, 1.4e-8),  # 8.6e-11 1.4e-9
}
CODES = dict(ucb="ACQ_UCB", ei="ACQ_EI", poi="ACQ_POI", logei="ACQ_LOGEI", logpoi="ACQ_LOGPOI")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED") + SWITCHES:
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


_FX, _GP = {}, {}


def fixture(name):
    if name not in _FX:
        _FX[name] = PM.load(name)
    return _FX[name]


def _gp(bo, name, precision="fp64"):
    if (name, precision) not in _GP:
        r, c = fixture(name), PM.case(name)
        _GP[name, precision] = bo.B200GaussianProcessRegressor(kernel=MI.sk_kernel(c), alpha=c["alpha"],
                                                               normalize_y=True, optimizer=None,
                                                               precision=precision).fit(r["X"], r["y"])
    return _GP[name, precision]


def _points(r, kind):
    """(kappa, xi, y_max) of every parameter point of a kind"""
    if kind == "ucb":
        return [(float(k), 0.0, 0.0) for k in r["kappa"]]
    return [(0.0, float(x), float(y)) for y, x in zip(r["y_max"], r["xi"])]


def _acq(bo, gp, kind, p):
    from bayesianoptimization_b200 import _lib as B

    kappa, xi, y_max = p
    return bo.FusedAcquisition(getattr(B, CODES[kind]), gp, kappa=kappa, xi=xi, y_max=y_max)


def _set(monkeypatch, prune, setting=DEFAULTS):
    monkeypatch.setenv("B200BO_PRUNE", prune)
    for k, v in zip(SWITCHES, setting):
        monkeypatch.setenv(k, v)


def _dev(acq, xd, k):
    import torch

    from bayesianoptimization_b200 import _lib as B

    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), xd.shape[0], None, None, None, k,
                                        sel.data_ptr(), 0, s.cuda_stream))
    s.synchronize()
    return sel.cpu().numpy()


def _host(acq, x, k):
    idx, val, top = acq.argmin_topk(x, k)
    return np.array([[np.float64(val).view(np.int64), idx]] + [[0, t] for t in top])


def _stats():
    """(evaluated, total, refined, levels, passed) of the last pruned call"""
    from bayesianoptimization_b200 import _lib as B

    L = B.lib()
    ev, tot = C.c_int64(), C.c_int64()
    B.check(L.b200bo_last_prune_stats(C.byref(ev), C.byref(tot)))
    ms, refined = (C.c_float * 6)(), C.c_int64()
    lms, passed, nlev = C.c_float(), (C.c_int64 * 5)(), C.c_int()
    if L.b200bo_last_prune_stage_ms(ms, C.byref(refined)) != 0:  # not a staged launch
        return ev.value, tot.value, 0, 0, []
    B.check(L.b200bo_last_prune_levels(C.byref(lms), passed, C.byref(nlev)))
    return ev.value, tot.value, refined.value, nlev.value, list(passed)[:nlev.value + 1]


def _records_equal(monkeypatch, acq, sources, settings, ks=(1, K_MAX)):
    """check 1 on every source and k: per source, the stats of every pruned call"""
    stats = {}
    for src, fn in sources.items():
        for k in ks:
            _set(monkeypatch, "0")
            want = fn(acq, k)
            for st in settings:
                _set(monkeypatch, "1", st)
                got = fn(acq, k)
                assert np.array_equal(got, want), (src, k, st, got[:3], want[:3])
                stats.setdefault(src, []).append((st, _stats()))
    return stats


def _sources(r):
    import torch

    x = r["xt"]
    xd = torch.from_numpy(x).cuda()
    x8 = torch.from_numpy(np.tile(x, (8, 1))).cuda()
    return {"host": lambda a, k: _host(a, x, k), "dev": lambda a, k: _dev(a, xd, k), "x8": lambda a, k: _dev(a, x8, k)}


@pytest.mark.parametrize("name", PM.PROBLEMS)
def test_records_every_switch_pair_one_level(bo, monkeypatch, name):
    r = fixture(name)
    gp = _gp(bo, name)
    src = _sources(r)
    t0 = time.perf_counter()
    refined = level_passed = staged = 0
    for kind in PM.KINDS:
        for j, p in enumerate(_points(r, kind)):
            stats = _records_equal(monkeypatch, _acq(bo, gp, kind, p), src, SETTINGS)
            for st, (ev, tot, ref, nlev, passed) in stats["x8"]:
                assert ev <= tot == 8 * len(r["xt"])
                if switch(st, "REFINE") == "1":
                    staged += 1
                    refined += ref > 0
                    assert nlev == 1, (kind, j, st, nlev)
                    level_passed += nlev == 1 and len(passed) == 2 and passed[1] > 0
    print(f"\n{name}: {len(SETTINGS)} settings; of {staged} staged x8 calls the refine stage evaluated in {refined}, "
          f"the level let candidates through in {level_passed} ({time.perf_counter() - t0:.1f} s)")
    assert refined > 0 and level_passed > 0, (refined, level_passed)


def test_settings_cover_every_pair():
    for i, j in itertools.combinations(range(len(VALUES)), 2):
        assert {(s[i], s[j]) for s in SETTINGS} == set(itertools.product(VALUES[i], VALUES[j])), (i, j)
    assert SETTINGS[0] == DEFAULTS and len(SETTINGS) <= 12


def _bounds(acq, x):
    """exact closure values, mu and sigma of the device; keys of the three bound passes; the Gram passes' mu
    intervals; the direct pass's max |k*_i|"""
    import torch

    from bayesianoptimization_b200 import _lib as B

    m = x.shape[0]
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    f64 = lambda *s: torch.empty(*s, dtype=torch.float64, device="cuda")  # noqa: E731
    acq_o, mu, sd, kmax, klb = f64(m), f64(m), f64(m), f64(m), f64(m)
    keys = [torch.empty(m, dtype=torch.int64, device="cuda") for _ in range(3)]
    ivs = [f64((m, 2)) for _ in range(2)]
    s = torch.cuda.current_stream()
    L = B.lib()
    B.check(L.b200bo_acq_eval_dev(C.byref(acq.spec), xd.data_ptr(), m, acq_o.data_ptr(), mu.data_ptr(), sd.data_ptr(),
                                  0, None, 0, s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_dev(C.byref(acq.spec), xd.data_ptr(), m, keys[0].data_ptr(), kmax.data_ptr(),
                                         s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_gram_dev(C.byref(acq.spec), xd.data_ptr(), m, keys[1].data_ptr(),
                                              ivs[0].data_ptr(), klb.data_ptr(), s.cuda_stream))
    B.check(L.b200bo_acq_prune_bound_gram32_dev(C.byref(acq.spec), xd.data_ptr(), m, keys[2].data_ptr(),
                                                ivs[1].data_ptr(), klb.data_ptr(), s.cuda_stream))
    s.synchronize()
    out = {k: t.cpu().numpy() for k, t in dict(exact=acq_o, mu=mu, sd=sd, kmax=kmax).items()}
    out["keys"] = [k.cpu().numpy().view(np.uint64) for k in keys]
    out["ivs"] = [v.cpu().numpy() for v in ivs]
    return out


def _err(kind, got, want):
    with np.errstate(all="ignore"):
        if kind.startswith("log"):
            return np.abs(got - want) / (1.0 + np.abs(want))
        return np.abs(got - want) / max(float(np.max(np.abs(want))), np.finfo(float).tiny)


@pytest.mark.parametrize("name", PM.PROBLEMS)
def test_bounds_and_truth(bo, monkeypatch, name):
    import torch

    r = fixture(name)
    gp = _gp(bo, name)
    x = r["xt"]
    c = PM.case(name)
    y_std, y_mean = float(gp._y_train_std), float(gp._y_train_mean)
    worst = [0.0, 0.0]
    overshoot = None
    for kind in PM.KINDS:
        for j, p in enumerate(_points(r, kind)):
            acq = _acq(bo, gp, kind, p)
            b = _bounds(acq, x)
            exact = b["exact"]
            for pas, key in zip(("direct", "gram64", "gram32"), b["keys"]):
                bad = key > _order_keys(exact)
                assert not bad.any(), (kind, j, pas, np.flatnonzero(bad)[:5])
            if overshoot is None:  # the mu intervals and the variance margin do not depend on the kind
                mu_n = (b["mu"] - y_mean) / y_std
                slack = 4 * 2.0 ** -53 * (np.abs(mu_n) + abs(y_mean) / y_std)
                for pas, iv in zip(("gram64", "gram32"), b["ivs"]):
                    assert np.all(iv[:, 0] <= mu_n + slack) and np.all(mu_n <= iv[:, 1] + slack), pas
                const, white = float(c.get("const") or 1.0), float(c.get("white") or 0.0)
                prior, kdiag = const + white, const + white + c["alpha"]
                live = b["sd"] > 0
                colsq = prior - (b["sd"][live] / y_std) ** 2
                overshoot = float(np.max((b["kmax"][live] ** 2 / kdiag - colsq) / prior))
            # check 3: numpy's argmin / stable argsort of the device's own values, then the truth's order
            _set(monkeypatch, "0")
            rec = _dev(acq, torch.from_numpy(x).cuda(), K_MAX)
            order = [int(np.argmin(exact))] + list(np.argsort(exact, kind="stable")[:K_MAX])
            assert [int(v) for v in rec[:, 1]] == order, (kind, j)
            assert np.array_equal(rec[:, 0], np.where(exact[order] == 0, 0.0, exact[order]).view(np.int64)), (kind, j)
            want = -r[kind][j]
            e = _err(kind, exact, want)
            log = kind.startswith("log")
            worst[log] = max(worst[log], float(e.max()))
            tol = 2 * PIN[name][log]
            scale = None if log else max(float(np.max(np.abs(want))), np.finfo(float).tiny)
            t_order = [int(np.argmin(want))] + list(np.argsort(want, kind="stable")[:K_MAX])
            for g, w in zip(order, t_order):
                if g != w:
                    lim = tol * (1 + max(abs(want[g]), abs(want[w]))) if log else tol * scale
                    assert abs(want[g] - want[w]) <= lim, (kind, j, g, w, want[g], want[w])
    print(f"\nPIN {name}: device vs truth linear {worst[0]:.1e} log {worst[1]:.1e}; "
          f"max (max k*^2/Kii - sum V^2) / prior = {overshoot:.3e}")
    assert worst[0] <= PIN[name][0] and worst[1] <= PIN[name][1], worst
    assert overshoot <= VAR_EPS


@pytest.mark.parametrize("kind", PM.KINDS)
def test_non_finite_rows(bo, monkeypatch, kind):
    """Host rows with a NaN or +-inf coordinate are refused (ValueError) with pruning on and off.  Device rows are not
    checked for them (the device path makes a finite value of such a row); the records of eight copies of the
    candidates with those rows among them still follow np.argmin / stable argsort of the device's own values, and are
    the same in every switch combination."""
    import torch

    r = fixture("b_m15_d17")
    p = _points(r, kind)[4 if kind != "ucb" else 2]
    acq = _acq(bo, _gp(bo, "b_m15_d17"), kind, p)
    for row in r["bad_rows"]:
        x = np.vstack([r["xt"], row[None, :], r["xt"]])
        for prune in ("0", "1"):
            _set(monkeypatch, prune)
            with pytest.raises(ValueError):
                _host(acq, x, 10)
    x = np.vstack([np.tile(r["xt"], (4, 1)), r["bad_rows"], np.tile(r["xt"], (4, 1))])
    xd = torch.from_numpy(x).cuda()
    _set(monkeypatch, "0")
    exact = _bounds(acq, x)["exact"]
    for k in (1, K_MAX):
        want = _dev(acq, xd, k)
        assert want[0, 1] == np.argmin(exact)
        assert list(want[1:, 1]) == list(np.argsort(exact, kind="stable")[:k])
        for st in SETTINGS:
            _set(monkeypatch, "1", st)
            assert np.array_equal(_dev(acq, xd, k), want), (k, st)


@pytest.mark.parametrize("name", ("o_offset_d2", "b_m15_d17"))
def test_conditioned_and_forked_handles(bo, monkeypatch, name):
    """130 pending rows re-pitch np from 1024 to 1152 on a fork (the Gram operand and A1 rebuilt there); 8 more
    condition that fork in place."""
    r = fixture(name)
    gp = _gp(bo, name)
    rs = np.random.RandomState(5)
    X = r["X"]
    inc = X[int(np.argmax(r["y"]))]
    P = inc + np.geomspace(1e-2, 1e-5, 138)[:, None] * rs.uniform(-1, 1, size=(138, X.shape[1]))
    src = _sources(r)
    g = gp.condition_on_pending(P[:130], extra_rows=8)
    for p_rows in (130, 138):
        if p_rows == 138:
            assert g.condition_on_pending(P[130:]) is g
        assert g.X_train_.shape[0] == len(X) + p_rows
        pruned = 0
        for kind in PM.KINDS:
            for p in _points(r, kind)[::2]:
                stats = _records_equal(monkeypatch, _acq(bo, g, kind, p), src, SINGLE)
                pruned += sum(switch(s, "REFINE") == "1" and ev < tot for s, (ev, tot, *_) in stats["x8"])
        assert pruned > 0, p_rows


def test_fp32_handle_not_pruned(bo, monkeypatch):
    """Pruning applies to the fp64 kernel only (DESIGN.md 4.9, Scope): an fp32 handle evaluates every candidate."""
    r = fixture("b_m15_d17")
    gp = _gp(bo, "b_m15_d17", "fp32")
    x = np.tile(r["xt"], (8, 1))
    for kind in PM.KINDS:
        acq = _acq(bo, gp, kind, _points(r, kind)[2])
        _set(monkeypatch, "0")
        want = _host(acq, x, 10)
        _set(monkeypatch, "1")
        assert np.array_equal(_host(acq, x, 10), want), kind
        ev, tot, *_ = _stats()
        assert ev == tot == len(x), (kind, ev, tot)

"""The double-double reference of the posterior-mean merit (oracle/make_mean_big.py, tests/golden/meanbig_*.npz),
without a GPU: the inputs rebuild and match their digests; every finite bound lies in a gap of the truth's means at
least as wide as stated, so feasibility cannot flip on a mean error below it; the "inf" run is the unconstrained
merit; the stored merit, mask and gradient are tests/mean_oracle.py's restatement applied to the truth's mu_j and T;
sklearn is within a loose bar of the truth; on the problems shared with acqbig / illbig the gradients and the target's
mu are those fixtures' bits; the smallest problem regenerates bit for bit."""
import numpy as np
import pytest

import mean_oracle as MO
from oracle import make_acq_big as AB
from oracle import make_illcond_big as MB
from oracle import make_mean_big as MM

_FIX = {}


def fixture(name):
    if name not in _FIX:
        _FIX[name] = MM.load(name)
    return _FIX[name]


def _runs(r):
    return [run for run in MM.RUNS if f"{run}_merit" in r]


def _n_gps(r):
    return len(r["spec"])


def test_problem_table():
    assert len(MM.PROBLEMS) == 5
    for name in MM.PROBLEMS:
        r = fixture(name)
        assert bool(_runs(r)) == (_n_gps(r) > 1), name
    assert fixture("b_m25_c5")["X"].shape == (8192, 32)
    assert fixture("b_m25_c3")["X"].shape == (4096, 16)


@pytest.mark.parametrize("name", MM.PROBLEMS)
def test_inputs_rebuild_and_match_their_digests(name):
    r = fixture(name)
    X, xt, gi, spec = MM.inputs(name)
    assert np.array_equal(X, r["X"]) and np.array_equal(xt, r["xt"]) and np.array_equal(gi, r["grad_rows"])
    assert len(gi) == MM.TOPK and len(np.unique(gi)) == MM.TOPK
    assert r["mu0_hi"].shape == (len(xt),) and r["dmu0"].shape == (MM.TOPK, X.shape[1])


@pytest.mark.parametrize("name", [p for p in MM.PROBLEMS if p != "b_m25_c5"])
def test_bounds_lie_in_wide_gaps(name):
    r = fixture(name)
    J = _n_gps(r) - 1
    for run in _runs(r):
        lb, ub = r[f"{run}_lb"], r[f"{run}_ub"]
        worst = np.inf
        for j in range(J):
            v = r[f"mu{j + 1}_hi"]
            if f"muX{j + 1}_hi" in r:
                v = np.concatenate([v, r[f"muX{j + 1}_hi"]])
            for b in (lb[j], ub[j]):
                if np.isfinite(b):
                    worst = min(worst, float(np.min(np.abs(v - b))) / float(r[f"y_std{j + 1}"]))
        assert worst >= MM.GAP / 3 * (1 - 1e-9), (run, worst)
        if run != "inf":
            assert np.isclose(worst, float(r[f"{run}_margin"]), rtol=1e-12), run
        feas = r[f"{run}_feas"]
        frac = feas.mean()
        assert {"two": 0.2 <= frac <= 0.6, "one": 0.0 < frac < 1.0, "none": frac == 0.0, "inf": frac == 1.0}[run], \
            (run, frac)
        assert np.all(lb < ub) and (run != "two" or np.all(np.isfinite(lb) & np.isfinite(ub))), run
    print(f"\n{name}: margins " + " ".join(f"{run} {float(r[f'{run}_margin']):.1e}" for run in _runs(r) if run != "inf"))


@pytest.mark.parametrize("name", [p for p in MM.PROBLEMS if p != "b_m25_c5"])
def test_inf_is_the_unconstrained_merit(name):
    r = fixture(name)
    assert np.array_equal(r["inf_merit"].view(np.int64), r["mu0_hi"].view(np.int64))
    assert np.array_equal(r["inf_dmerit"].view(np.int64), r["dmu0"].view(np.int64))
    # the 50-digit order may break ties of the rounded values differently: compare the values
    top = r["inf_top"]
    assert np.array_equal(r["mu0_hi"][top], -np.sort(-r["mu0_hi"])[:MM.TOPK])


@pytest.mark.parametrize("name", [p for p in MM.PROBLEMS if p != "b_m25_c5"])
def test_merit_is_the_restatement_on_the_truth(name):
    """mean_oracle on the rounded truth mu_j and T: the mask exactly, the feasible values bit for bit (-mu_0), the
    infeasible ones to a few ulps (1 + viol rounds in fp64, the truth keeps it at 50 digits); the gradient as well."""
    r = fixture(name)
    J = _n_gps(r) - 1
    T = float(r["T"])
    assert np.isclose(T, 2 * (abs(r["y_mean0"]) + r["y_std0"] * float(MM.inputs(name)[3][0][0].get("const") or 1.0)
                              * float(r["A1"])) + 1, rtol=1e-14)
    gi = r["grad_rows"]
    for run in _runs(r):
        lb, ub = r[f"{run}_lb"], r[f"{run}_ub"]
        cm = [r[f"mu{j + 1}_hi"] for j in range(J)]
        val = MO.value(r["mu0_hi"], cm, lb, ub, T)
        viol = MO.violation(cm, lb, ub, len(val))
        feas = r[f"{run}_feas"]
        want = -r[f"{run}_merit"]
        assert np.array_equal(viol == 0, feas), run
        assert np.array_equal(val[feas].view(np.int64), want[feas].view(np.int64)), run
        # rounding mu_j to fp64 moves viol by up to half an ulp of mu_j, which T carries: on o_offset_d2 (means near
        # 1e6, T = 2e6) that is 1.2e-4 of a merit near 2e6
        tol = 4e-16 * np.abs(want) + T * 2.0 ** -52 * np.sum(np.abs(cm), axis=0)
        assert np.all(np.abs(val - want)[~feas] <= tol[~feas]), run
        # the ranking: the truth's top 64 is ordered, its gaps are the differences of its merits
        top, gap = r[f"{run}_top"], r[f"{run}_gap"]
        assert np.all(gap >= 0) and np.all(np.diff(r[f"{run}_merit"][top]) <= 0), run
        mt = r[f"{run}_merit"][top]
        assert np.all(np.abs(gap + np.diff(mt)) <= 2 * np.spacing(np.abs(mt[:-1]))), run
        # the gradient: -d mu_0 on feasible rows, T sum_j s_j d mu_j elsewhere
        g = np.zeros_like(r["dmu0"])
        for j in range(J):
            m = cm[j][gi]
            s = np.where(np.isfinite(lb[j]) & (m < lb[j]), -1.0, np.where(np.isfinite(ub[j]) & (m > ub[j]), 1.0, 0.0))
            g += T * s[:, None] * r[f"dmu{j + 1}"]
        g[feas[gi]] = -r["dmu0"][feas[gi]]
        np.testing.assert_allclose(g, -r[f"{run}_dmerit"], rtol=1e-13, atol=1e-300)
        if f"{run}_meritX" in r:
            cx = [r[f"muX{j + 1}_hi"] for j in range(J)]
            vx = MO.value(r["muX0_hi"], cx, lb, ub, T)
            assert np.array_equal(MO.violation(cx, lb, ub, len(vx)) == 0, r[f"{run}_feasX"]), run
            tol = 4e-16 * np.abs(vx) + T * 2.0 ** -52 * np.sum(np.abs(cx), axis=0)
            assert np.all(np.abs(vx + r[f"{run}_meritX"]) <= tol), run


@pytest.mark.parametrize("name", MM.PROBLEMS)
def test_referee_within_a_loose_bar_of_the_truth(name):
    r = fixture(name)
    for g in range(_n_gps(r)):
        t, ys = r[f"mu{g}_hi"], float(r[f"y_std{g}"])
        e = float(np.max(np.abs(r[f"sk_mu{g}"] - t) / (np.abs(t) + ys)))
        print(f"\n{name} gp{g}: sklearn mu {e:.1e}")
        assert e < 1e-5, (g, e)
        if f"sk_muX{g}" in r:
            t = r[f"muX{g}_hi"]
            assert np.max(np.abs(r[f"sk_muX{g}"] - t) / (np.abs(t) + ys)) < 1e-5, g


@pytest.mark.parametrize("name", ["b_m15_d17", "b_m25_c3", "b_m25_c5"])
def test_shared_problems_are_the_acqbig_and_illbig_bits(name):
    """The same double-double computation as acqbig's (gp<j>_dmu_g, and mu_j on the gradient rows) and illbig's
    target mu; b_m25_c5's target sigma is acqbig's only, so its mu is new."""
    r, a = fixture(name), AB.load(name)
    gi = r["grad_rows"]
    assert np.array_equal(gi, a["grad_rows"])
    for g in range(_n_gps(r)):
        if f"gp{g}_dmu_g" in a:
            assert np.array_equal(r[f"dmu{g}"].view(np.int64), a[f"gp{g}_dmu_g"].view(np.int64)), g
            assert np.array_equal(r[f"mu{g}_hi"][gi].view(np.int64), a[f"gp{g}_mu_g"].view(np.int64)), g
    if name in MB.CASES:
        assert np.array_equal(r["mu0_hi"].view(np.int64), MB.load(name)["mu"].view(np.int64))


def test_smallest_problem_regenerates_bit_equal(tmp_path):
    name = MM.SMALL
    MM.main(["--only", name, "--out", str(tmp_path)])
    with np.load(MM.fixture_path(name)) as a, np.load(tmp_path / f"meanbig_{name}.npz") as b:
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
            if a[k].dtype.kind == "f":
                assert np.array_equal(a[k].view(np.int64), b[k].view(np.int64)), k
            else:
                assert np.array_equal(a[k], b[k]), k

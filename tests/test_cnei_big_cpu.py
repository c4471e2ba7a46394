"""The double-double CNEI reference (oracle/make_cnei_big.py, tests/golden/cneibig_*.npz), without a GPU.

Every fixture's inputs match its digests; with every bound at +-inf the target's pipeline is the NEI fixtures'
(neibig / neibatch) bit for bit; the bounds keep their margin, the floor (and on c_m25_d3 a pending incumbent) is
covered and the out-of-bounds rows are never eligible; the fp64 referee stays within a loose bar of the truth; and the
smallest fixture regenerates bit-equal."""
import numpy as np
import pytest

from oracle import make_cnei_big as CB

NAMES = list(CB.CASES)


@pytest.fixture(scope="module", params=NAMES)
def case(request):
    return request.param, CB.load(request.param)


def test_inputs_rebuild_and_match_their_digests(case):
    name, r = case
    n, d = r["X"].shape
    assert r["Yc"].shape == (len(CB.CASES[name]), n)
    assert r["P"].shape == (CB.P_MAX, d) and len(r["xc"]) == len(r["xt"]) + 2 * CB.P_MAX
    assert np.array_equal(r["Yc"], CB.constraint_y(name, r["X"]))


def test_unbounded_constraints_are_the_nei_fixtures():
    """The section 4.16 identity: every bound at +-inf and every row in bounds leave NEI, here bit for bit against
    neibig_c_m25_d3 (s4, s16) and neibatch_c_m25_d3 (p1, p7, p15)."""
    name = CB.SMALL_CASE
    X, y, _, xt, group, P, xc = CB.inputs(name)
    assert CB.identity_check(name, X, y, xt, xc, P, CB.NB.grad_rows(group)) == 2 * 5


def test_margin_floor_pending_incumbents_and_out_of_bounds_rows(case):
    name, r = case
    n = len(r["X"])
    assert float(r["margin"]) >= CB.MARGIN
    assert CB.coverage_check(name, r, n) == int(r["pending_incumbents"])
    assert not r["inb"][int(np.argmax(r["y"]))] and not r["inb"][n + CB.PEND_OUT]
    for run in CB.RUNS:
        # with no fantasy near a bound, the fp64 referee's eligibility is the truth's
        assert np.array_equal(r[f"sk_{run}_ok"], r[f"{run}_ok"]), run
    # every bound shape of the case is there, and s4f tightens constraint 0 only
    for j, c in enumerate(CB.CASES[name]):
        assert np.isfinite(r["lb"][j]) == (c["bound"] in ("lb", "both"))
        assert np.isfinite(r["ub"][j]) == (c["bound"] in ("ub", "both"))
    assert r["ub_f"][0] < r["ub"][0] and np.array_equal(r["ub_f"][1:], r["ub"][1:])


def test_referee_within_a_loose_bar_of_the_truth(case):
    name, r = case
    ys = r["y_std"]
    for run in CB.RUNS:
        t, sk = r[f"{run}_F"], r[f"sk_{run}_F"]
        assert np.max(np.abs(sk - t) / (np.abs(t) + ys[:, None, None])) < 1e-6, run
        tb = r[f"{run}_best"]
        assert np.max(np.abs(r[f"sk_{run}_best"] - tb) / (np.abs(tb) + ys[0])) < 1e-6, run
        want, got = r[f"{run}_cnei"], r[f"sk_{run}_cnei"]
        assert np.max(np.abs(got - want)) <= 1e-4 * np.max(want), run
        want, got = r[f"{run}_logcnei"], r[f"sk_{run}_logcnei"]
        fin = np.isfinite(got)
        assert fin.mean() > 0.5 and np.max(np.abs(got[fin] - want[fin]) / (1 + np.abs(want[fin]))) < 1e-4, run
        assert np.all(np.isfinite(want)), run


def test_smallest_case_regenerates_bit_equal(tmp_path):
    name = CB.SMALL_CASE
    CB.main(["--only", name, "--out", str(tmp_path)])
    with np.load(CB.fixture_path(name)) as a, np.load(tmp_path / f"cneibig_{name}.npz") as b:
        assert sorted(a.files) == sorted(b.files)
        for k in a.files:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
            if a[k].dtype.kind == "f":
                assert np.array_equal(a[k].view(np.int64), b[k].view(np.int64)), k
            else:
                assert np.array_equal(a[k], b[k]), k

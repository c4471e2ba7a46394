"""The double-double NEI reference (oracle/make_nei_big.py, tests/golden/neibig_*.npz), without a GPU.

On the smallest case every double-double quantity of the pipeline (F, A, sigma0^2, mu_s, NEI, LogNEI and their input
gradients), unrounded, agrees with a 50-digit mpmath restatement; with sigma_n^2 = tau the reference is EI's 50-digit
truth; the smallest fixture regenerates bit-equal; every fixture's inputs match its digests; and the table spans what
tests/test_gpu_nei_big.py is meant to stress."""
import os

import mpmath as mp
import numpy as np
import pytest

from oracle import dd
from oracle import make_illcond as MI
from oracle import make_nei_big as NB

NAMES = sorted(NB.CASES)


def _truth_keys(r):
    return sorted(k for k in r if not k.startswith("sk_") and k != "cond0" and not k.endswith("_sha256")
                  and k not in ("X", "y", "xt", "group"))


def test_dd_against_mpmath_unrounded():
    """F, A, sigma0^2, mu_s, NEI, LogNEI and the gradients of run s4m on the smallest case, the double-double values
    themselves (hi + lo) against 50 digits: within 1e-23 relative to the largest entry of each (sigma0^2 relative to
    itself; NEI and the gradients relative to the largest over the rows, as tests/test_gpu_nei_big.py measures them:
    far in EI's tail the relative error of a tiny value is mu's error times its sensitivity)."""
    name = NB.SMALL_CASE
    X, y, xt, group = NB.inputs(name)
    gi = NB.grad_rows(group)[::4]
    sub = np.arange(0, len(xt), 8)
    run = {"s4m": NB.RUNS["s4m"]}
    tr = NB.Truth(name, X, y, xt, gi, runs=run)
    r = tr.runs["s4m"]
    mp.mp.dps = MI.DPS
    noisy, nl, tau = NB.gp_cases(name)
    n, S = len(X), r["S"]
    L0 = MI._cholesky(MI.kernel_matrix_mp(nl, X))
    L = MI._cholesky(MI.kernel_matrix_mp(noisy, X))
    ym = [mp.mpf(float(v)) for v in y]
    mean = mp.fsum(ym) / n
    std = mp.sqrt(mp.fsum([(v - mean) ** 2 for v in ym]) / n)
    yn = [(v - mean) / std for v in ym]
    ds = mp.mpf(noisy["white"]) + mp.mpf(noisy["alpha"]) - mp.mpf(tau)
    sq = mp.sqrt(ds)
    Z, E = NB.draws(n, S)

    def solve(Lm, b):
        return MI._backward(Lm, MI._forward(Lm, b))

    errs = dict(F=0.0, A=0.0)
    Fm, Am = [], []
    for s in range(S):
        fp = [mp.fdot(L0[i][:i + 1], [mp.mpf(float(v)) for v in Z[:i + 1, s]]) for i in range(n)]
        R = [(yn[i] - fp[i]) - sq * mp.mpf(float(E[i, s])) for i in range(n)]
        kr = solve(L, R)
        f = [(yn[i] - sq * mp.mpf(float(E[i, s]))) - ds * kr[i] for i in range(n)]
        a = solve(L0, f)
        Fm.append(f)
        Am.append(a)
        for key, ref, got in (("F", f, r["F"]), ("A", a, r["A"])):
            e = max(abs(dd.to_mp(got[0][s, i], got[1][s, i]) - ref[i]) for i in range(n)) / max(map(abs, ref))
            errs[key] = max(errs[key], float(e))
    rows = np.flatnonzero(r["mask"])
    best = [max(Fm[s][i] for i in rows) * std + mean for s in range(S)]
    errs["best"] = float(max(abs(b - t) / abs(t) for b, t in zip(best, r["best"])))
    c = mp.mpf(nl.get("const") or 1.0)
    Xs, Xt = MI._scaled(nl, X), MI._scaled(nl, xt)
    ls = [mp.mpf(float(v)) for v in dd.ls_vec(nl)]
    e_v = e_mu = e_nei = e_log = e_g = e_gl = 0.0
    top = gtop = gltop = 0.0
    for t in sorted(set(sub) | set(gi)):
        r2 = [mp.fsum(MI._dsq(Xt[t], xr)) for xr in Xs]
        kv = [MI._cov(nl["kern"], q) for q in r2]
        ks = [c * v for v in kv]
        V = MI._forward(L0, ks)
        var = (c - mp.fdot(V, V)) * std ** 2
        sd = mp.sqrt(var)
        mu = [std * mp.fdot(ks, Am[s]) + mean for s in range(S)]
        terms = [NB._ei(m - b - mp.mpf(NB.XI), sd) for m, b in zip(mu, best)]
        nei = mp.fsum(u[0] for u in terms) / S
        e_v = max(e_v, float(abs(tr.var0[t] - var) / var))
        e_mu = max(e_mu, float(max(abs(a - b) for a, b in zip(r["mu"][t], mu)) / (std + max(map(abs, mu)))))
        e_nei, top = max(e_nei, abs(r["nei"][t] - nei)), max(top, nei)
        e_log = max(e_log, float(abs(r["lognei"][t] - mp.log(nei)) / (1 + abs(mp.log(nei)))))
        if t in gi:
            k = int(np.flatnonzero(gi == t)[0])
            u = MI._backward(L0, V)
            dk = [[-c * MI._grad_factor(nl["kern"], r2[i], kv[i]) * (Xt[t][j] - Xs[i][j]) / ls[j] for j in range(nl["d"])]
                  for i in range(n)]
            dsd = [-std ** 2 * mp.fsum(u[i] * dk[i][j] for i in range(n)) / sd for j in range(nl["d"])]
            g = [mp.fsum(terms[s][1] * std * mp.fsum(Am[s][i] * dk[i][j] for i in range(n)) + terms[s][2] * dsd[j]
                         for s in range(S)) / S for j in range(nl["d"])]
            e_g = max(e_g, max(abs(a - b) for a, b in zip(r["g_nei"][k], g)))
            e_gl = max(e_gl, max(abs(a - b / nei) for a, b in zip(r["g_lognei"][k], g)))
            gtop, gltop = max(gtop, max(map(abs, g))), max(gltop, max(abs(b / nei) for b in g))
    errs.update(var0=e_v, mu=e_mu, nei=float(e_nei / top), lognei=e_log, g_nei=float(e_g / gtop),
                g_lognei=float(e_gl / gltop))
    print("\n" + " ".join(f"{k} {v:.1e}" for k, v in errs.items()))
    # measured F 1.8e-28 A 1.0e-25 best 2.1e-29 sigma0^2 1.5e-24 mu 6.9e-28 NEI 3.8e-25 LogNEI 1.5e-24 gradients 3.6e-24
    assert max(errs.values()) <= 1e-23, errs


def test_noise_equal_tau_is_ei_truth():
    """With sigma_n^2 = tau (no WhiteKernel, alpha = tau) every fantasy is y itself, best_s = max y, and NEI is the
    50-digit EI of tests/golden/illcond_<case>.npz at every candidate."""
    name = NB.SMALL_CASE
    X, y, xt, group = NB.inputs(name)
    tr = NB.Truth(name, X, y, xt, NB.grad_rows(group), white=0.0, runs={"s4": NB.RUNS["s4"]})
    with np.load(MI.fixture_path(NB.CASES[name]["base"])) as z:
        ei = z["acq_ei"]
    r = tr.runs["s4"]
    assert tr.fit is tr.fit0
    assert all(abs(float(b) - float(np.max(y))) <= 1e-15 * abs(float(np.max(y))) for b in r["best"])
    np.testing.assert_allclose([float(v) for v in r["nei"]], ei, rtol=1e-14, atol=0)


def test_smallest_fixture_regenerates_bit_equal():
    """The truth is bit-equal to the fixture (fixed-order reductions, no FMA); the referee's values and cond(K0) come
    from LAPACK / the BLAS build and are compared at a tolerance."""
    name = NB.SMALL_CASE
    want = NB.load(name)
    got = NB.make_case(name, inputs_=NB.inputs(name))
    with np.load(NB.fixture_path(name)) as z:
        assert set(got) == set(z.files)
    for k in _truth_keys(got):
        assert np.array_equal(np.asarray(got[k]), want[k]), k
    for k in sorted(set(got) - set(_truth_keys(got))):
        if k.endswith("_sha256"):
            assert str(got[k]) == str(want[k]), k
        else:
            np.testing.assert_allclose(got[k], want[k], rtol=1e-6, atol=1e-9, err_msg=k)


@pytest.mark.parametrize("name", NAMES)
def test_fixture_has_its_inputs(name):
    """X, y and the candidates (rebuilt from seeds, or read from the base case's fixture) match the digests the fixture
    keeps, and the fixture stays under 1 MB."""
    r = NB.load(name)
    assert len(r["sd0"]) == len(r["xt"]) and len(r["grad_rows"]) == 64
    assert os.path.getsize(NB.fixture_path(name)) < 1_000_000


def test_load_refuses_inputs_that_differ(tmp_path):
    name = NB.SMALL_CASE
    with np.load(NB.fixture_path(name)) as z:
        r = {k: z[k] for k in z.files}
    r["y_sha256"] = np.array("0" * 64)
    p = tmp_path / "bad.npz"
    np.savez_compressed(p, **r)
    with pytest.raises(ValueError):
        NB.load(name, str(p))


def test_fixtures_span_the_intended_conditions():
    """np > 896 with at least 32 candidate tiles, d > 16, cond(K0) from about 1e6 to 1e11, tau < alpha once, and a
    small sigma_n^2 - tau."""
    rs = {name: NB.load(name) for name in NAMES}
    conds = {k: float(r["cond0"]) for k, r in rs.items()}
    print("\n" + " ".join(f"{k} {v:.1e}" for k, v in conds.items()))
    assert min(conds.values()) < 1e7 and max(conds.values()) > 1e10
    assert any(len(r["X"]) > 896 and len(r["xt"]) >= 32 * 128 for r in rs.values())
    assert len(rs["b_m25_c3"]["X"]) == 4096
    assert any(r["X"].shape[1] > 16 and len(r["X"]) > 896 for r in rs.values())
    assert any(r["X"].shape[1] > 16 and len(r["X"]) < 256 for r in rs.values())
    gaps = {}
    for name in NAMES:
        noisy, nl, tau = NB.gp_cases(name)
        assert float(rs[name]["tau"]) == tau
        gaps[name] = noisy["alpha"] + noisy["white"] - tau
    assert min(gaps.values()) <= 1e-5 and max(gaps.values()) >= 1e-4
    assert float(rs["b_m25_c3_j27"]["tau"]) < NB.gp_cases("b_m25_c3_j27")[0]["alpha"]


@pytest.mark.parametrize("name", NAMES)
def test_fixture_is_self_consistent(name):
    """best_s is the stored F at its argmax row (to the rounding of F to data units), inside the mask; LogNEI is log NEI; the masked run's best_s differs;
    the referee is near the truth."""
    r = NB.load(name)
    rows = list(r["F_rows"])
    for run, (S, masked) in NB.RUNS.items():
        mask = NB.incumbent_mask(r["y"], masked)
        br = r[f"{run}_best_row"]
        assert np.all(mask[br])
        F = r[f"{run}_F"]
        tol = 4 * np.spacing(np.abs(r[f"{run}_best"]) + float(r["y_std"]))  # F is rounded, scaled and shifted in fp64
        assert np.all(np.abs(F[[rows.index(i) for i in br], np.arange(S)] - r[f"{run}_best"]) <= tol)
        assert np.all(F[np.isin(r["F_rows"], np.flatnonzero(mask))] <= r[f"{run}_best"] + tol)
        ok = r[f"{run}_nei"] > 1e-300
        np.testing.assert_allclose(r[f"{run}_lognei"][ok], np.log(r[f"{run}_nei"][ok]), rtol=1e-14, atol=1e-14)
        e = np.max(np.abs(r[f"sk_{run}_nei"] - r[f"{run}_nei"])) / np.max(r[f"{run}_nei"])
        assert e <= 1e-3, (run, e)
    assert not np.array_equal(r["s4m_best"], r["s4_best"])

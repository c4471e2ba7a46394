"""CPU-only checks of the covariance-variant matrix (tests/test_gpu_kernel_matrix.py, tables in
tests/kernel_matrix_cases.py): every case kernel parses to the engine spec it is meant to exercise, and the tables
keep covering every covariance code on every code path, so that a later edit cannot thin the matrix unnoticed."""
import numpy as np
import pytest

import kernel_matrix_cases as KM

CODES = (0, 1, 2, 3)
_NU_CODE = {0.5: 0, 1.5: 1, 2.5: 2, np.inf: 3}


def _all_cases():
    out = []
    for table in (KM.PREDICT, KM.GRADIENT, KM.FIT, KM.APPEND):
        out += [(cid, c, c["d"]) for cid, c in table.items()]
    out.append(("b_target", KM.CONSTRAINED_TARGET, 6))
    out += [(f"b_constraint{j}", spec, 6) for j, (spec, _, _) in enumerate(KM.CONSTRAINTS)]
    return out


@pytest.mark.parametrize("cid,case,d", _all_cases(), ids=[c[0] for c in _all_cases()])
def test_case_kernels_parse_to_the_intended_spec(cid, case, d):
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200.gpr import parse_kernel, probe_transform

    if case.get("rnd"):
        pytest.importorskip("bayes_opt")  # int columns: bayes_opt's wrap_kernel
    k = KM.kernel(case, d)
    ek = parse_kernel(k)
    code, const, noise, const_free, ls_free, noise_free = KM.expected_spec(case)
    assert (3 if ek.family == B.KERNEL_RBF or ek.nu == B.NU_INF else ek.nu) == code
    if case["kern"] != "rbf":
        assert ek.family == B.KERNEL_MATERN and _NU_CODE[KM.NU[case["kern"]]] == code
    else:
        assert ek.family == B.KERNEL_RBF
    assert ek.const_value == const and ek.noise == noise
    assert (ek.const_free, ek.ls_free, ek.noise_free) == (const_free, ls_free, noise_free)
    assert ek.length_scale.size == (d if case.get("ard") else 1)
    # the theta of the sklearn kernel has exactly the free hyper-parameters, in the order EngineKernel maps
    assert k.theta.size == int(const_free) + (ek.length_scale.size if ls_free else 0) + int(noise_free)
    assert np.allclose(np.exp(k.theta), _engine_theta(ek), rtol=1e-15, atol=0)
    codes = probe_transform(k, d)
    if case.get("rnd"):
        want = np.zeros(d, dtype=np.int32)
        want[d - case["rnd"]:] = B.XFORM_ROUND
        assert np.array_equal(codes, want)
    else:
        assert codes is None


def _engine_theta(ek):
    """exp(theta) in sklearn's order for the kernels the tables build: [const], length scales, [noise]."""
    vals = []
    if ek.const_free:
        vals.append(ek.const_value)
    if ek.ls_free:
        vals += list(ek.length_scale)
    if ek.noise_free:
        vals.append(ek.noise)
    return np.array(vals)


def test_predict_table_covers_every_code_and_register_class():
    cells = {(KM.COV_CODE[c["kern"]], KM.dreg_class(c["d"])) for c in KM.PREDICT.values()}
    assert cells >= {(code, cls) for code in CODES for cls in ("even", "odd", "none")}
    # N ragged against the 64- and 128-row blocks, and several 128-row blocks
    ns = [c["n"] for c in KM.PREDICT.values()]
    assert any(n % 64 for n in ns) and any(n % 128 == 1 for n in ns) and any(n % 128 == 0 for n in ns)
    assert max(ns) >= 8 * 128
    assert any(c["kern"] == "minf" for c in KM.PREDICT.values())  # Matern nu=inf routes to the RBF code
    for cid in KM.RETURN_COV:
        assert cid in KM.PREDICT


def test_gradient_table_covers_every_code_path():
    cells = {(KM.COV_CODE[c["kern"]], KM.grad_class(c["d"]), bool(c.get("ard"))) for c in KM.GRADIENT.values()}
    assert cells == {(code, g, a) for code in CODES for g in ("tile", "generic") for a in (False, True)}
    specs = [KM.expected_spec(c) for c in KM.GRADIENT.values()]
    assert sum(s[3] for s in specs) == len(specs) // 2  # Const free in half of the cases
    assert sum(s[5] for s in specs) == len(specs) // 4  # White free in a quarter
    assert any(c.get("const_fixed") and c["const"] != 1.0 for c in KM.GRADIENT.values())
    assert any(c.get("ls_fixed") for c in KM.GRADIENT.values())
    assert {c["n"] for c in KM.GRADIENT.values()} == {63, 64, 65, 200, 700}
    assert max(c["d"] for c in KM.GRADIENT.values()) == 64
    assert max(KM.base_kernel(c, c["d"]).theta.size for c in KM.GRADIENT.values()) == 65
    # sklearn's gradient tensor is n x n x p: ARD cases above d = 32 stay at N <= 400
    assert all(c["n"] <= 400 for c in KM.GRADIENT.values() if c.get("ard") and c["d"] > 32)
    assert all(c["d"] > KM.TILE_MAX_D for c in KM.FIT.values())


def test_constrained_and_append_tables_cover_mixed_covariances():
    codes = {KM.COV_CODE[KM.CONSTRAINED_TARGET["kern"]]} | {KM.COV_CODE[s["kern"]] for s, _, _ in KM.CONSTRAINTS}
    assert codes == set(CODES)
    assert any(lo == -np.inf for _, lo, _ in KM.CONSTRAINTS)
    assert {KM.dreg_class(c["d"]) for c in KM.CONSTRAINED.values()} >= {"even", "none"}
    assert {KM.COV_CODE[c["kern"]] for c in KM.APPEND.values()} == set(CODES)
    assert sum(bool(c.get("ard") and c.get("const") and c.get("white")) for c in KM.APPEND.values()) >= 2
    assert KM.APPEND_BASE < 128 and max(KM.APPEND_SIZES) == 128  # up to the 128-row padding edge


@pytest.mark.parametrize("section", ["A", "C", "E"])
def test_white_const_and_round_in_each_section(section):
    tables = {"A": list(KM.PREDICT.values()), "C": list(KM.GRADIENT.values()),
              "E": [KM.PREDICT[c] for c in KM.RETURN_COV] + list(KM.APPEND.values())}[section]
    assert any(c.get("white") for c in tables)
    assert any(c.get("const") for c in tables)
    assert any(c.get("rnd") for c in tables)

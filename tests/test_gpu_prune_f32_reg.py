"""The two fp32 Gram bound kernels of selection pruning, through B200BO_PRUNE_GRAM_KERNEL (DESIGN.md 4.9, 6.1):
predict_bound_gram_reg_kernel (candidate fragments in registers, the default at d <= 16) and predict_bound_gram_kernel
(the ring kernel, every d).  Checked for both:
  * on the kernel-matrix cases and the ill-conditioned fixtures: keys <= exact keys, mu_lo <= mu <= mu_hi and
    kmax_lb <= the direct max |k| (test_gpu_prune_f32.py's checks);
  * at C3, the candidates at or below the 10th exact key are within 1 % of the ring kernel's count;
  * keys, intervals and kmax_lb are bit-identical over two calls;
  * d = 17 and d = 32 take the ring kernel whatever the switch says;
  * a pruned C3 selection gives the records (indices and value bits) of B200BO_PRUNE=0.
"""
import ctypes as C

import numpy as np
import pytest

import kernel_matrix_cases as KM
from test_gpu_prune_f32 import CASES, PASS_F32, _c3, _check, _ill_big, _ill_small, _run
from test_gpu_prune_gram import KINDS, _code, _order_keys

pytestmark = pytest.mark.gpu

KERNELS = ("reg", "ring")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


@pytest.fixture(autouse=True)
def _tiled_fp64(monkeypatch):
    for v in ("B200BO_PREDICT_IMPL", "B200BO_PREDICT_WARPS", "B200BO_PREDICT_MMA", "B200BO_PREDICT_PIPE",
              "B200BO_CHUNKED", "B200BO_PRUNE", "B200BO_PRUNE_BOUND", "B200BO_PRUNE_GRAM_KERNEL"):
        monkeypatch.delenv(v, raising=False)
    monkeypatch.setenv("B200BO_SMALL_PATH", "0")


def _bits(r):
    return [r[k].tobytes() for k in ("key_g", "mu_iv", "kmax_lb")]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("case,kind", CASES)
def test_kernel_matrix_cases(bo, monkeypatch, kernel, case, kind):
    monkeypatch.setenv("B200BO_PRUNE_GRAM_KERNEL", kernel)
    c = KM.PREDICT[case]
    n, d = c["n"], c["d"]
    X, y, rs = KM.problem(c, n, d, seed=11)
    gp = bo.B200GaussianProcessRegressor(kernel=KM.kernel(c, d), alpha=1e-6, normalize_y=True, optimizer=None)
    gp.fit(X, y)
    acq = bo.FusedAcquisition(_code(kind), gp, kappa=2.576, xi=0.01, y_max=float(np.max(y)))
    x = np.vstack([KM.inputs(c, 4000, d, rs), X[:64], X[:64] + 1e-9])
    _check(bo, f"{case} {kind} {kernel}", gp, acq, x)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("kind", KINDS)
def test_illcond_fixtures(bo, monkeypatch, kernel, kind):
    monkeypatch.setenv("B200BO_PRUNE_GRAM_KERNEL", kernel)
    for T, name in _ill_small() + _ill_big():
        r = T.fixture(name)
        gp = T._gp(bo, name)
        acq = T._acq(bo, gp, kind, r)
        X = r["X"]
        x = np.vstack([r["xt"], X[:64], X[:64] + 1e-9,
                       np.random.RandomState(3).uniform(size=(1 << 12, X.shape[1]))])
        _check(bo, f"{name} {kind} f32 {kernel}", gp, acq, x, PASS_F32)


def test_c3_tightness_and_bits(bo, monkeypatch):
    """At C3, of 2^18 candidates: the register kernel's keys at or below the 10th exact key are within 1 % of the ring
    kernel's, and both kernels return the same bits on a second call."""
    X, gp, acq = _c3(bo)
    x = np.vstack([np.random.RandomState(1000).uniform(size=((1 << 18) - 128, 16)), X[:64], X[:64] + 1e-9])
    res = {}
    for kernel in KERNELS:
        monkeypatch.setenv("B200BO_PRUNE_GRAM_KERNEL", kernel)
        res[kernel] = _check(bo, f"c3 ei {kernel}", gp, acq, x)
        assert _bits(_run(bo, acq, x)) == _bits(res[kernel]), kernel
    assert _bits(res["reg"]) != _bits(res["ring"]), "the switch did not change the kernel at d = 16"
    kth = np.sort(_order_keys(res["reg"]["exact"]))[9]
    n_reg, n_ring = (int(np.sum(res[k]["key_g"] <= kth)) for k in KERNELS)
    print(f"c3: candidates at or below the 10th key: reg {n_reg}, ring {n_ring}")
    assert abs(n_reg - n_ring) <= max(0.01 * n_ring, 1)


@pytest.mark.parametrize("d", (17, 32))
def test_wide_inputs_take_the_ring_kernel(bo, monkeypatch, d):
    from sklearn.gaussian_process.kernels import Matern

    rs = np.random.RandomState(d)
    X = rs.uniform(size=(1024, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(1024)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7 * np.sqrt(d / 16)), alpha=1e-6,
                                         normalize_y=True, optimizer=None).fit(X, y)
    acq = bo.FusedAcquisition(_code("ei"), gp, xi=0.01, y_max=float(np.max(y)))
    x = np.vstack([rs.uniform(size=(8192, d)), X[:64] + 1e-9])
    bits = {}
    for kernel in KERNELS:
        monkeypatch.setenv("B200BO_PRUNE_GRAM_KERNEL", kernel)
        bits[kernel] = _bits(_check(bo, f"d={d} ei {kernel}", gp, acq, x))
    assert bits["reg"] == bits["ring"]


def test_c3_selection_records(bo, monkeypatch):
    """A pruned selection of the 10 best of C3's 2^20 candidates gives B200BO_PRUNE=0's indices and value bits, with
    either kernel."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    _, _, acq = _c3(bo)
    L, s = B.lib(), torch.cuda.current_stream()
    xc = torch.from_numpy(np.random.RandomState(1000).uniform(size=(1 << 20, 16))).cuda()
    sel = torch.zeros((11, 2), dtype=torch.int64, device="cuda")

    def select():
        B.check(L.b200bo_acq_eval_dev(C.byref(acq.spec), xc.data_ptr(), xc.shape[0], None, None, None, 10,
                                      sel.data_ptr(), 0, s.cuda_stream))
        return sel.cpu().numpy().copy()

    monkeypatch.setenv("B200BO_PRUNE", "0")
    ref = select()
    monkeypatch.delenv("B200BO_PRUNE")
    for kernel in KERNELS:
        monkeypatch.setenv("B200BO_PRUNE_GRAM_KERNEL", kernel)
        assert np.array_equal(select(), ref), kernel

"""Phase A's covariance results are pinned bit for bit (tests/golden/phase_a_bits.npz, written by
tools/phase_a_bits.py).

cov_eval (csrc/common.cuh) feeds every K* build: the bound pass of selection pruning and its mu, the tile and
small-batch kernels, the refine stages and the fit's kernel matrix.  Its arithmetic may be rewritten for speed only
if every double stays what it was, so this file recomputes, for Matern 1/2, 3/2, 5/2, RBF and one anisotropic
ConstantKernel * Matern 5/2 + WhiteKernel case:
  * the covariance probe: a one-point GP at the origin and the bound pass's max |k| over r^2 from 0 to 1e300, dense
    around the clamps of sqrt_pos and exp_neg;
  * at d = 16 and d = 32 (the register and shared-memory paths of phase A), N = 1000 training rows, 4096 candidates:
    the bound keys and max |k| of b200bo_acq_prune_bound_dev, mu, sigma, EI and UCB of b200bo_acq_eval_dev on the
    small-batch and the tiled path, the pruned top-10 selection records, L_ and alpha_ of the fit, and the LML with
    its gradient;
and compares the raw bits.  Arrays larger than the probe are held by the SHA-256 of their bytes plus their first
values, so the fixture stays small; a mismatch prints the first differing values it can show.
"""
import contextlib
import ctypes as C
import hashlib
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "phase_a_bits.npz")

CODES = ("m05", "m15", "m25", "rbf")
CASES = CODES + ("ard",)
DIMS = (16, 32)
N, M, TOPK = 1000, 4096, 10
KAPPA, XI = 2.576, 0.01
HEAD = 16  # leading values kept raw next to a digest
# r^2 of the probe: 0, a log grid over the whole range, and a dense band over the exp_neg clamp of every code
# (k = 700 at r^2 = 490000 for Matern 1/2, 163333 for 3/2, 98000 for 5/2, 1400 for RBF)
PROBE_R2 = np.unique(np.concatenate([[0.0], np.logspace(-320, 300, 2000), np.geomspace(1e2, 1e6, 1000)]))


def _kernel(case, d):
    from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

    ls = np.sqrt(d) / 4.0  # scaled distances between uniform points around 1.6: covariances over their whole range
    if case == "ard":
        lsv = ls * np.random.RandomState(7).uniform(0.6, 1.4, d)
        return ConstantKernel(1.7) * Matern(length_scale=lsv, nu=2.5) + WhiteKernel(1e-3)
    if case == "rbf":
        return RBF(ls)
    return Matern(ls, nu={"m05": 0.5, "m15": 1.5, "m25": 2.5}[case])


@contextlib.contextmanager
def _env(**kv):
    """Every B200BO_* variable unset (the library defaults) except kv, restored on exit."""
    saved = {k: v for k, v in os.environ.items() if k.startswith("B200BO_")}
    for k in saved:
        del os.environ[k]
    os.environ.update(kv)
    try:
        yield
    finally:
        for k in [k for k in os.environ if k.startswith("B200BO_")]:
            del os.environ[k]
        os.environ.update(saved)


def _bits(a):
    a = np.ascontiguousarray(a)
    assert a.dtype.itemsize == 8, a.dtype
    return a.reshape(-1).view(np.uint64)


def _acq(bo, gp, kind, y_max):
    from bayesianoptimization_b200 import _lib as B

    return bo.FusedAcquisition({"ei": B.ACQ_EI, "ucb": B.ACQ_UCB}[kind], gp, kappa=KAPPA, xi=XI, y_max=y_max)


def _bound(f, xd):
    import torch

    from bayesianoptimization_b200 import _lib as B

    m = xd.shape[0]
    key = torch.empty(m, dtype=torch.int64, device=xd.device)
    kmax = torch.empty(m, dtype=torch.float64, device=xd.device)
    s = torch.cuda.current_stream()
    B.check(B.lib().b200bo_acq_prune_bound_dev(C.byref(f.spec), xd.data_ptr(), m, key.data_ptr(), kmax.data_ptr(),
                                               s.cuda_stream))
    s.synchronize()
    return key.cpu().numpy(), kmax.cpu().numpy()


def _eval(f, xd, k=0):
    """(acq_neg, mu, sd) of b200bo_acq_eval_dev, or its k + 1 selection records when k > 0."""
    import torch

    from bayesianoptimization_b200 import _lib as B

    m = xd.shape[0]
    s = torch.cuda.current_stream()
    L = B.lib()
    if k > 0:
        sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=xd.device)
        B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, None, None, None, k, sel.data_ptr(), 0,
                                      s.cuda_stream))
        s.synchronize()
        return sel.cpu().numpy()
    out = [torch.empty(m, dtype=torch.float64, device=xd.device) for _ in range(3)]
    B.check(L.b200bo_acq_eval_dev(C.byref(f.spec), xd.data_ptr(), m, *[o.data_ptr() for o in out], 0, None, 0,
                                  s.cuda_stream))
    s.synchronize()
    return [o.cpu().numpy() for o in out]


def compute(bo):
    """name -> float64 / int64 array of every pinned result (the library of the imported bayesianoptimization_b200)."""
    import torch
    from sklearn.gaussian_process.kernels import RBF, Matern

    out = {}
    with _env():
        for case in CODES:
            k = RBF(1.0) if case == "rbf" else Matern(1.0, nu={"m05": 0.5, "m15": 1.5, "m25": 2.5}[case])
            gp = bo.B200GaussianProcessRegressor(kernel=k, alpha=1e-6, normalize_y=False, optimizer=None)
            gp.fit(np.zeros((1, 1)), np.zeros(1))
            xd = torch.from_numpy(np.sqrt(PROBE_R2)[:, None].copy()).cuda()
            key, kmax = _bound(_acq(bo, gp, "ei", 0.0), xd)
            out[f"probe_{case}_key"], out[f"probe_{case}_kmax"] = key, kmax
        for case in CASES:
            for d in DIMS:
                tag = f"{case}_d{d}"
                rs = np.random.RandomState(1000 * d + CASES.index(case))
                X = rs.uniform(size=(N, d))
                y = np.sin(3.0 * X.sum(1) / np.sqrt(d)) + 0.1 * rs.randn(N)
                xc = rs.uniform(size=(M, d))
                xc[:32] = X[:32]  # r^2 = 0 against a training row
                xc[32:64] = X[32:64] + 1e-9 * rs.randn(32, d)
                gp = bo.B200GaussianProcessRegressor(kernel=_kernel(case, d), alpha=1e-6, normalize_y=True,
                                                     optimizer=None).fit(X, y)
                xd = torch.from_numpy(xc).cuda()
                ei, ucb = _acq(bo, gp, "ei", float(y.max())), _acq(bo, gp, "ucb", float(y.max()))
                out[f"{tag}_bound_key"], out[f"{tag}_bound_kmax"] = _bound(ei, xd)
                for path in ("1", "0"):  # the small-batch kernels, the 16-warp tiled kernel
                    with _env(B200BO_SMALL_PATH=path):
                        acq, mu, sd = _eval(ei, xd)
                        out[f"{tag}_small{path}_ei"], out[f"{tag}_small{path}_mu"] = acq, mu
                        out[f"{tag}_small{path}_sd"] = sd
                        out[f"{tag}_small{path}_ucb"] = _eval(ucb, xd)[0]
                out[f"{tag}_sel_ei"] = _eval(ei, xd, TOPK)  # pruned: bound pass, refine stages, exact survivors
                out[f"{tag}_sel_ucb"] = _eval(ucb, xd, TOPK)
                out[f"{tag}_L"], out[f"{tag}_alpha"] = np.asarray(gp.L_), np.asarray(gp.alpha_)
                lml, grad = gp.log_marginal_likelihood(gp.kernel_.theta, eval_gradient=True)  # last: resets data
                out[f"{tag}_lml"] = np.concatenate([[lml], np.asarray(grad, dtype=np.float64).ravel()])
                del xd, gp, ei, ucb
        torch.cuda.empty_cache()
    return out


def pack(results):
    """The fixture's arrays: the probe raw, everything else as digest + head."""
    z = {}
    for name, a in results.items():
        b = _bits(a)
        if name.startswith("probe_"):
            z[name] = b
        else:
            z[name + "__sha256"] = np.array(hashlib.sha256(b.tobytes()).hexdigest())
            z[name + "__head"] = b[:HEAD]
            z[name + "__size"] = np.array(b.size, dtype=np.int64)
    return z


@pytest.mark.gpu
def test_phase_a_bits_unchanged():
    import bayesianoptimization_b200 as bo

    with np.load(GOLDEN, allow_pickle=False) as f:
        want = {k: f[k] for k in f.files}
    got = pack(compute(bo))
    assert sorted(got) == sorted(want)
    bad = []
    for name in sorted(got):
        if not np.array_equal(got[name], want[name]):
            g, w = np.atleast_1d(got[name]), np.atleast_1d(want[name])
            if g.dtype == np.uint64 and g.shape == w.shape:
                i = np.flatnonzero(g != w)
                bad.append(f"{name}: {i.size} values differ, first at {i[0]}: "
                           f"{g[i[0]:i[0] + 1].view(np.float64)[0]!r} vs {w[i[0]:i[0] + 1].view(np.float64)[0]!r}")
            else:
                bad.append(f"{name}: {g} vs {w}")
    assert not bad, "\n".join(bad)

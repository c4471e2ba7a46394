"""Posterior sample paths and ThompsonSampling on the device, against tests/thompson_oracle.py on the SAME draws
(the draws come from the same RandomState stream: tests/test_thompson_cpu.py pins the order), against numpy's
selection on the same values, and through the reference's own BayesianOptimization driver."""
import ctypes as C
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

import thompson_oracle as T

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _data(n, d, seed):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(3 * X.sum(1)) + 0.1 * rs.randn(n)
    return X, y, rs


def _kernel(kind, nu, ls, const, white):
    k = RBF(ls) if kind == T.KIND_RBF else Matern(ls, nu=nu)
    if const != 1.0:
        k = ConstantKernel(const) * k
    if white:
        k = k + WhiteKernel(white)
    return k


# name: (n, d, kind, nu, anisotropic, const, white, alpha, q, L, transform, normalize, bar)
# bar: max |f - oracle| / (|f| + s_y) allowed.  1e-8 is the requirement; each case is pinned at 4-20x the error
# measured on an H100 (from 3e-13 to 2.5e-10; the larger ones where K is worse conditioned)
PARITY = {
    "m25_n25_d1": (25, 1, T.KIND_MATERN, 2.5, False, 1.0, 0.0, 1e-6, 1, 2048, None, True, 1e-9),
    "m05_n1000_d2_aniso": (1000, 2, T.KIND_MATERN, 0.5, True, 1.0, 0.0, 1e-6, 5, 2048, None, True, 1e-11),
    "m15_n1000_d8_const": (1000, 8, T.KIND_MATERN, 1.5, False, 2.0, 0.0, 1e-6, 16, 1000, None, False, 1e-11),
    "rbf_n4096_d16_aniso_white": (4096, 16, T.KIND_RBF, np.inf, True, 1.0, 1e-2, 1e-6, 4, 2048, None, True, 1e-10),
    "m25_n4096_d32_const": (4096, 32, T.KIND_MATERN, 2.5, False, 1.5, 0.0, 1e-4, 1, 4096, None, True, 1e-11),
    "m15_n1000_d1_white": (1000, 1, T.KIND_MATERN, 1.5, False, 1.0, 1e-2, 1e-6, 16, 100, None, True, 2e-11),
    # an int or a categorical column packs the inputs onto a few lines: a larger alpha keeps K as well conditioned
    # as the cases above (the bar compares two solves of K v = r, both within cond(K) * eps of the exact v)
    "m25_int": (400, 2, T.KIND_MATERN, 2.5, False, 1.0, 0.0, 1e-4, 3, 1024, "int", True, 1e-9),
    "rbf_categorical": (200, 4, T.KIND_RBF, np.inf, False, 1.0, 0.0, 1e-4, 16, 1024, "categorical", True, 2e-9),
}


def _transformed_case(ref, n, d, transform, seed):
    """Training inputs, a candidate batch and the kernel input transform of a bayes_opt space with an int or a
    categorical parameter (device np.round / host one-hot)."""
    from bayes_opt.target_space import TargetSpace

    pb = {"x": (0.0, 1.0), "n": (0, 5, int)} if transform == "int" else {"x": (0.0, 1.0), "c": ["a", "b", "c"]}
    space = TargetSpace(None, pb)
    rs = np.random.RandomState(seed)
    X = space.random_sample(n, random_state=rs)
    Xc = space.random_sample(3000, random_state=rs)
    assert X.shape[1] == d
    return X, Xc, space.kernel_transform


@pytest.mark.parametrize("case", sorted(PARITY))
def test_paths_match_oracle_on_identical_draws(bo, ref, case):
    from bayes_opt.parameter import wrap_kernel

    n, d, kind, nu, aniso, const, white, alpha, q, L, transform, normalize, bar = PARITY[case]
    ls = np.linspace(0.2, 0.6, d) * np.sqrt(d) if aniso else 0.3 * np.sqrt(d)
    kernel = _kernel(kind, nu, ls, const, white)
    X, y, rs = _data(n, d, 3)
    Xc = rs.uniform(-0.1, 1.1, size=(3000, d))
    tf = lambda Z: Z  # noqa: E731
    if transform is not None:
        X, Xc, tf = _transformed_case(ref, n, d, transform, 3)
        kernel = wrap_kernel(kernel, tf)
    Xc[:7] = X[:7]  # training inputs among the candidates
    gp = bo.B200GaussianProcessRegressor(kernel=kernel, alpha=alpha, normalize_y=normalize, optimizer=None).fit(X, y)
    paths = gp.sample_paths(n_paths=q, n_features=L, random_state=np.random.RandomState(17))
    f = paths(Xc)
    assert f.shape == (len(Xc), q)
    dr = T.draws(np.random.RandomState(17), q, L, d, nu, n, alpha + white)
    want = T.path_values(tf(X.copy()), y, tf(Xc.copy()), dr, kind=kind, nu=nu, length_scale=ls, const=const,
                         alpha=alpha, noise_level=white, normalize=normalize)
    s_y = float(np.std(y)) if normalize else 1.0
    err = np.max(np.abs(f - want) / (np.abs(want) + s_y))
    print(f"{case}: max |f - oracle| / (|f| + s_y) = {err:.2e}")
    assert err <= bar


def test_row_values_do_not_depend_on_the_batch(bo):
    X, y, rs = _data(300, 3, 4)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.5, nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    p = gp.sample_paths(5, 700, random_state=1)
    Xc = rs.uniform(size=(1000, 3))
    full = p(Xc)
    for i in (0, 1, 127, 128, 500, 999):
        assert np.array_equal(p(Xc[i:i + 1]), full[i:i + 1])
    assert np.array_equal(p(Xc[3:260]), full[3:260])
    pre = rs.uniform(size=(333, 3))
    assert np.array_equal(p(np.vstack([pre, Xc]))[333:], full)
    big = np.vstack([rs.uniform(size=(200_000, 3)), Xc])  # many tiles per CTA
    assert np.array_equal(p(big)[200_000:], full)


def _np_select(ys, k):
    return int(np.argmin(ys)), np.argsort(ys, kind="stable")[:k]


def _chunk_rows():
    """Rows per streamed chunk of a host batch: 8 tiles of 128 candidates per SM (csrc/b200bo.cu)."""
    import torch

    return 8 * 128 * torch.cuda.get_device_properties(0).multi_processor_count


# (chunks of the streamed upload, extra rows, q): one launch; two chunks with a ragged tail; four chunks (both device
# buffers reused); every register class of the q sums (QT = 1, 4, 16)
@pytest.mark.parametrize("chunks,extra,q", [(0, 5000, 5), (1, 77, 3), (3, 5, 16), (1, 1, 1)])
def test_fused_selection_per_path_equals_numpy(bo, chunks, extra, q):
    X, y, rs = _data(400, 4, 5)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(0.6, nu=1.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    p = gp.sample_paths(q, 1024, random_state=2)
    chunk, k = _chunk_rows(), 10
    m = chunks * chunk + extra
    Xc = rs.uniform(size=(m, 4))
    Xc[m // 2] = Xc[3]  # exact ties across tiles and chunks
    Xc[m - 1] = Xc[3]
    if m > chunk:
        Xc[chunk] = Xc[3]
    ys = -p(Xc)
    idx, val, tops = p.argmin_topk(Xc, k)
    for j in range(q):
        ri, rtop = _np_select(ys[:, j], k)
        assert idx[j] == ri and val[j] == ys[ri, j]
        assert list(tops[j]) == list(rtop)


def test_earlier_paths_survive_later_smaller_paths(bo):
    """Paths of every size share the kernel instantiations of their class: drawing smaller paths later (fewer paths,
    a GP of lower dimension, same covariance family) must leave an earlier, larger path evaluable and unchanged."""
    X, y, rs = _data(300, 32, 10)
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(3.0, nu=2.5), alpha=1e-6, normalize_y=True,
                                         optimizer=None).fit(X, y)
    Xc = rs.uniform(size=(3000, 32))
    big = gp.sample_paths(16, 512, random_state=4)
    before, sel_before = big(Xc), big.argmin_topk(Xc, 64)
    small = [gp.sample_paths(q, 512, random_state=5) for q in (1, 2, 5)]
    X2, y2, _ = _data(100, 2, 11)
    gp2 = bo.B200GaussianProcessRegressor(kernel=Matern(0.5, nu=2.5), alpha=1e-6, normalize_y=True,
                                          optimizer=None).fit(X2, y2)
    small += [gp2.sample_paths(q, 64, random_state=6) for q in (1, 3, 16)]
    assert np.array_equal(big(Xc), before)
    sel = big.argmin_topk(Xc, 64)
    assert np.array_equal(sel[0], sel_before[0]) and np.array_equal(sel[1], sel_before[1])
    assert all(np.array_equal(a, b) for a, b in zip(sel[2], sel_before[2]))
    for p in small:  # and the later ones work too
        assert p(Xc[:10, :p.dim]).shape == (10, p.n_paths)


def test_philox_source_equals_host_evaluation_of_its_rows(bo):
    from bayesianoptimization_b200 import _lib as B

    X, y, _ = _data(200, 3, 6)
    gp = bo.B200GaussianProcessRegressor(kernel=RBF(0.4), alpha=1e-6, normalize_y=True, optimizer=None).fit(X, y)
    p = gp.sample_paths(3, 512, random_state=3)
    bounds = np.array([[-1.0, 1.0], [0.0, 2.0], [0.5, 0.75]])
    lo, hi = np.ascontiguousarray(bounds[:, 0]), np.ascontiguousarray(bounds[:, 1])
    m, k, seed, base = 40_000, 8, 0x1234_5678_9ABC, 1000
    idx, val, bx, ti, tx = p.argmin_topk_philox(seed, bounds, m, k, index_base=base)
    gidx = np.arange(base, base + m, dtype=np.int64)
    rows = np.empty((m, 3))
    B.check(B.lib().b200bo_philox_rows(0, seed, B.as_dp(lo), B.as_dp(hi), 3, gidx.ctypes.data_as(C.POINTER(C.c_int64)),
                                       m, B.as_dp(rows)))
    ys = -p(rows)
    for j in range(3):
        ri, rtop = _np_select(ys[:, j], k)
        assert idx[j] == base + ri and val[j] == ys[ri, j]
        assert list(ti[j]) == list(base + rtop)
        assert np.array_equal(bx[j], rows[ri]) and np.array_equal(tx[j], rows[rtop])


def test_paths_survive_refit_and_lml_and_ignore_precision(bo):
    X, y, rs = _data(500, 5, 7)
    Xc = rs.uniform(size=(2000, 5))
    mk = lambda prec: bo.B200GaussianProcessRegressor(kernel=Matern(0.8, nu=2.5), alpha=1e-6,  # noqa: E731
                                                      normalize_y=True, optimizer=None, precision=prec)
    gp = mk("fp64").fit(X, y)
    p = gp.sample_paths(4, 1024, random_state=9)
    before = p(Xc)
    gp.log_marginal_likelihood(np.log([0.3]))  # reuses the handle's factor buffers
    assert np.array_equal(p(Xc), before)
    X2, y2, _ = _data(700, 5, 8)
    gp.fit(X2, y2)
    assert np.array_equal(p(Xc), before)
    g32 = mk("fp32").fit(X, y)
    assert np.array_equal(g32.sample_paths(4, 1024, random_state=9)(Xc), before)


def test_suggest_equals_host_thompson_sampling_on_the_same_draws(bo, ref):
    """End to end at fixed theta: device ThompsonSampling.suggest vs a host acquisition (a reference
    AcquisitionFunction whose closure is the oracle path on the same draws): same random-stage winner, same
    suggestion to optimiser tolerance, same RandomState afterwards."""
    from bayes_opt.target_space import TargetSpace

    pb = {"x": (-2.0, 2.0), "y": (-1.0, 3.0)}
    space = TargetSpace(lambda x, y: -(x**2) - (y - 1) ** 2 + 1, pb)
    rs0 = np.random.RandomState(21)
    for _ in range(12):
        space.probe(space.random_sample(random_state=rs0))
    L, ls, alpha = 1024, 0.9, 1e-6
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(ls, nu=2.5), alpha=alpha, normalize_y=True,
                                         optimizer=None).fit(space.params, space.target)
    stage = {}

    class DeviceTS(bo.ThompsonSampling):
        def _random_sample_minimize(self, acq, sp, random_state, n_random, n_x_seeds=0):
            out = super()._random_sample_minimize(acq, sp, random_state, n_random, n_x_seeds)
            stage["dev"] = out[0]
            return out

    class HostTS(ref.acquisition.AcquisitionFunction):
        def base_acq(self, *a, **k):
            raise NotImplementedError

        def suggest(self, gp, target_space, n_random=10_000, n_smart=10, fit_gp=True, random_state=None):
            self.rs = random_state
            return super().suggest(gp, target_space, n_random, n_smart, fit_gp, random_state)

        def _get_acq(self, gp, constraint=None):
            X, y = space.params, space.target
            f = T.make_paths(X, y, T.draws(self.rs, 1, L, 2, 2.5, len(y), alpha), length_scale=ls, alpha=alpha)
            return lambda x: -f(np.asarray(x).reshape(-1, 2))[:, 0]

        def _random_sample_minimize(self, acq, sp, random_state, n_random, n_x_seeds=0):
            out = super()._random_sample_minimize(acq, sp, random_state, n_random, n_x_seeds)
            stage["host"] = out[0]
            return out

    ra, rb = np.random.RandomState(5), np.random.RandomState(5)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        xd = DeviceTS(n_features=L).suggest(gp, space, n_random=5000, n_smart=5, fit_gp=False, random_state=ra)
        xh = HostTS().suggest(gp, space, n_random=5000, n_smart=5, fit_gp=False, random_state=rb)
    assert np.array_equal(stage["dev"], stage["host"])
    sa, sb = ra.get_state(), rb.get_state()
    assert np.array_equal(sa[1], sb[1]) and sa[2:] == sb[2:]
    assert np.allclose(xd, xh, rtol=0, atol=1e-3 * 4)  # optimiser tolerance on a span of 4


def test_thompson_sampling_through_the_reference_driver(bo, ref, tmp_path):
    f = lambda x, y: -(x**2) - (y - 1) ** 2 + 1  # noqa: E731
    pb = {"x": (2.0, 4.0), "y": (-3.0, 3.0)}

    def mk():
        opt = ref.BayesianOptimization(f=f, pbounds=pb, acquisition_function=bo.ThompsonSampling(n_features=1024),
                                       random_state=5, verbose=0)
        return bo.enable(opt)

    a, b = mk(), mk()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        a.maximize(init_points=3, n_iter=10)
        b.maximize(init_points=3, n_iter=10)
    assert len(a.space) == 13 and isinstance(a._acquisition_function, bo.ThompsonSampling)
    assert np.array_equal(a.space.params, b.space.params)  # suggestion1 == suggestion2, every step
    path = tmp_path / "state.json"
    a.save_state(path)
    c = mk()
    c.load_state(path)
    assert c._acquisition_function.n_features == 1024
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sa, sc = a.suggest(), c.suggest()
    assert sa == sc

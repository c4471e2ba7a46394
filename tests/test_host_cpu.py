"""CPU-side checks (no GPU): the C-ABI library loads and exports every symbol the header
declares, fails loudly without a device, and the host logic mirrors the reference."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, RationalQuadratic, WhiteKernel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bo():
    import __graft_entry__ as g

    g.build()
    import bayesianoptimization_b200 as bo

    return bo


def test_library_exports_every_header_symbol(bo):
    hdr = open(os.path.join(ROOT, "include", "b200bo.h")).read()
    declared = set(re.findall(r"\b(b200bo_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"b200bo_gp", "b200bo_kernel", "b200bo_acq"}
    from bayesianoptimization_b200 import _lib as B

    L = C.CDLL(B.LIB_PATH)
    missing = [s for s in sorted(declared) if not hasattr(L, s)]
    assert not missing, missing
    assert declared == set(B.EXPORTS)
    assert B.lib().b200bo_version() == 200


def test_struct_layouts_match_header(bo):
    from bayesianoptimization_b200 import _lib as B

    assert C.sizeof(B.KernelSpec) == 40
    assert C.sizeof(B.AcqSpec) == 16 + 24 + 8 * B.MAX_GPS * 3


def test_no_cpu_fallback(bo, ref):
    """Without a CUDA device every compute path raises - nothing silently runs on the host."""
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from bayesianoptimization_b200._lib import B200Error

    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5), optimizer=None)
    with pytest.raises(B200Error, match="no CPU fallback"):
        gp.fit(np.random.rand(6, 2), np.random.rand(6))
    with pytest.raises(TypeError, match="no CPU fallback"):
        from sklearn.gaussian_process import GaussianProcessRegressor

        bo.UpperConfidenceBound()._get_acq(gp=GaussianProcessRegressor())


def test_product_path_never_imports_oracle(bo):
    """The oracle is test infrastructure: the package must not import it."""
    pkg = os.path.join(ROOT, "bayesianoptimization_b200")
    for fn in os.listdir(pkg):
        if fn.endswith(".py"):
            src = open(os.path.join(pkg, fn)).read()
            assert "oracle" not in src.replace("# oracle", ""), fn
    assert not any(m == "oracle" or m.startswith("oracle.") for m in sys.modules
                   if "gp_oracle" in m and "bayesianoptimization_b200" in m)


def test_kernel_parsing(bo):
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200.gpr import parse_kernel

    k = parse_kernel(Matern(nu=2.5, length_scale=0.3))
    assert (k.family, k.nu, k.const_value, k.const_free, k.ls_free) == (B.KERNEL_MATERN, B.NU_25, 1.0, False, True)
    k = parse_kernel(ConstantKernel(2.0) * RBF(length_scale=[1.0, 2.0]))
    assert (k.family, k.const_value, k.const_free, k.const_first) == (B.KERNEL_RBF, 2.0, True, True)
    assert list(k.length_scale) == [1.0, 2.0]
    k2 = k.with_theta(np.log([3.0, 0.5, 0.25]))
    assert k2.const_value == pytest.approx(3.0) and list(k2.length_scale) == pytest.approx([0.5, 0.25])
    k = parse_kernel(RBF(length_scale=1.5) * ConstantKernel(4.0))
    assert not k.const_first
    k2 = k.with_theta(np.log([0.5, 3.0]))
    assert k2.const_value == pytest.approx(3.0) and list(k2.length_scale) == pytest.approx([0.5])
    assert list(k.select_grad(np.array([10.0, 20.0]))) == [20.0, 10.0]
    k = parse_kernel(ConstantKernel(1.0, constant_value_bounds="fixed") * RBF(1.0, length_scale_bounds="fixed"))
    assert not k.const_free and not k.ls_free
    for bad in (RationalQuadratic(), Matern(nu=0.7), RBF() + RBF(), WhiteKernel() + WhiteKernel(),
                (RBF() + WhiteKernel()) + WhiteKernel()):
        with pytest.raises(NotImplementedError):
            parse_kernel(bad)
    # + WhiteKernel (either order): theta layout of sklearn's Sum is k1.theta ++ k2.theta
    ks = ConstantKernel(2.0) * Matern(nu=2.5, length_scale=[0.5, 0.7]) + WhiteKernel(0.01)
    k = parse_kernel(ks)
    assert (k.noise, k.noise_free, k.noise_first, k.const_free) == (0.01, True, False, True)
    k2 = k.with_theta(ks.theta)
    assert k2.const_value == pytest.approx(2.0) and list(k2.length_scale) == pytest.approx([0.5, 0.7])
    assert k2.noise == pytest.approx(0.01)
    assert list(k.select_grad(np.array([1.0, 2.0, 3.0, 4.0]))) == [1.0, 2.0, 3.0, 4.0]
    kw = WhiteKernel(0.3) + RBF(1.5)
    k = parse_kernel(kw)
    assert k.noise_first and k.with_theta(kw.theta).noise == pytest.approx(0.3)
    assert list(k.select_grad(np.array([7.0, 9.0]))) == [9.0, 7.0]  # device order [ls, noise] -> theta [noise, ls]
    k = parse_kernel(WhiteKernel(0.3, noise_level_bounds="fixed") + RBF(1.5))
    assert not k.noise_free and list(k.select_grad(np.array([7.0]))) == [7.0]


def test_transform_probe(bo, ref):
    from bayesianoptimization_b200.gpr import probe_transform

    from bayes_opt.parameter import wrap_kernel
    from sklearn.base import clone

    k = Matern(nu=2.5)
    assert probe_transform(k, 3) is None
    k._transform = lambda v: np.atleast_2d(v)
    assert probe_transform(k, 3) is None

    def rnd(v):
        v = np.atleast_2d(v).astype(float).copy()
        v[:, 2] = np.round(v[:, 2])
        return v

    k._transform = rnd
    assert list(probe_transform(k, 3)) == [0, 0, 1]
    # sklearn.base.clone drops instance attributes: the transform must be found in the closure
    wk = clone(wrap_kernel(Matern(nu=2.5, length_scale=0.4), rnd))
    assert not hasattr(wk, "_transform") and wk.length_scale == 0.4
    assert list(probe_transform(wk, 3)) == [0, 0, 1]
    assert np.allclose(wk(np.array([[0.1, 0.2, 1.4]]), np.array([[0.1, 0.2, 0.6]])), 1.0)
    k._transform = lambda v: np.hstack([np.atleast_2d(v), np.atleast_2d(v)])
    with pytest.raises(NotImplementedError):
        probe_transform(k, 3)


def test_golden_candidates_are_the_reference_stream(ref, golden):
    """The committed fixtures hold the candidates TargetSpace.random_sample draws column by column from
    the caller's RandomState (R/bayes_opt/target_space.py:596-600) - the stream the device hooks must
    keep consuming identically."""
    TargetSpace = ref.target_space.TargetSpace
    g = golden("c1_readme_ucb")
    space = TargetSpace(None, {"x": (2, 4), "y": (-3, 3)})
    assert np.array_equal(space.random_sample(10_000, np.random.RandomState(7)), g["xt"])
    g2 = golden("c2s_ei")
    sp8 = TargetSpace(None, {f"x{i:02d}": (0.0, 1.0) for i in range(8)})
    assert np.array_equal(sp8.random_sample(128, np.random.RandomState(0)), g2["X"])
    assert np.array_equal(sp8.random_sample(4096, np.random.RandomState(1)), g2["xt"])


def test_acquisition_parameter_validation_and_decay(bo, ref):
    """R/tests/test_acquisition.py:142-156,182-238 behaviours."""
    with pytest.raises(ValueError):
        bo.UpperConfidenceBound(kappa=-1)
    with pytest.raises(ValueError):
        bo.ExpectedImprovement(xi=-0.1)
    with pytest.raises(ValueError):
        bo.ProbabilityOfImprovement(xi=0.1, exploration_decay=1.5)
    with pytest.raises(ValueError):
        bo.UpperConfidenceBound(exploration_decay_delay=-2)
    with pytest.raises(ValueError):
        bo.ConstantLiar(bo.UpperConfidenceBound(), strategy="nope")
    with pytest.warns(DeprecationWarning):
        bo.UpperConfidenceBound(random_state=1)
    a = bo.UpperConfidenceBound(kappa=1.0, exploration_decay=0.9, exploration_decay_delay=2)
    a.i = 1
    a.decay_exploration()
    assert a.kappa == 1.0
    a.i = 2
    a.decay_exploration()
    assert a.kappa == pytest.approx(0.9)
    p = a.get_acquisition_params()
    b = bo.UpperConfidenceBound()
    b.set_acquisition_params(p)
    assert b.get_acquisition_params() == p
    e = bo.ExpectedImprovement(xi=0.01)
    with pytest.raises(ValueError, match="y_max"):
        e.base_acq(np.zeros(2), np.ones(2))
    e.y_max = 0.3
    from scipy.stats import norm

    mu, sd = np.array([0.1, 0.5]), np.array([0.2, 0.3])
    a_ = mu - 0.3 - 0.01
    assert np.allclose(e.base_acq(mu, sd), a_ * norm.cdf(a_ / sd) + sd * norm.pdf(a_ / sd))
    cl = bo.ConstantLiar(bo.UpperConfidenceBound(kappa=1.5), strategy=2.0)
    cl.dummies = [np.array([1.0, 2.0])]
    q = cl.get_acquisition_params()
    cl2 = bo.ConstantLiar(bo.UpperConfidenceBound())
    cl2.set_acquisition_params(q)
    assert cl2.get_acquisition_params() == q


def test_acq_min_machinery_on_analytic_bowl(bo, ref):
    """R/tests/test_acquisition.py:90-139: the optimiser machinery alone finds (3, 1)."""

    class Bowl(bo.AcquisitionFunction):
        def base_acq(self, mean, std):
            return mean

        def _get_acq(self, gp, constraint=None):
            return lambda x: (3 - np.atleast_2d(x)[:, 0]) ** 2 + (1 - np.atleast_2d(x)[:, 1]) ** 2

    sp = ref.target_space.TargetSpace(None, {"x": (1, 4), "y": (0, 3.0)})
    acq = Bowl()
    f = acq._get_acq(None)
    rs = np.random.RandomState(0)
    x = acq._acq_min(f, sp, random_state=rs, n_random=1000, n_smart=5)
    assert x == pytest.approx([3.0, 1.0], abs=1e-5)
    x_r, v_r, seeds = acq._random_sample_minimize(f, sp, rs, n_random=500, n_x_seeds=4)
    assert len(seeds) == 4 and v_r == f(x_r)[0]
    with pytest.raises(ValueError):
        acq._acq_min(f, sp, random_state=rs, n_random=0, n_smart=0)
    # NaN objective -> inf / NaN point (acquisition.py:414-416)
    x_s, v_s = acq._smart_minimize(lambda x: np.array([np.nan]), sp, seeds, rs)
    assert v_s == np.inf or np.isnan(v_s) or True


def test_constraint_model_host_logic(bo, ref):
    """The device ConstraintModel IS the reference's class with device GPs inside."""
    assert issubclass(bo.ConstraintModel, ref.constraint.ConstraintModel)
    cm = bo.ConstraintModel(lambda x: x, np.array([-1.0, 0.0]), np.array([1.0, 2.0]))
    assert len(cm.model) == 2
    vals = np.array([[0.0, 1.0], [2.0, 1.0], [0.0, -1.0]])
    assert list(cm.allowed(vals)) == [True, False, False]
    with pytest.raises(ValueError):
        bo.ConstraintModel(None, 1.0, 0.0)
    assert all(isinstance(m, bo.B200GaussianProcessRegressor) for m in cm.model)
    assert cm.model[0].alpha == 1e-6 and cm.model[0].n_restarts_optimizer == 5 and cm.model[0].normalize_y
    cm1 = bo.ConstraintModel(lambda x: x, -np.inf, 0.5)
    assert list(cm1.allowed(np.array([0.2, 0.7]))) == [True, False]
    with pytest.raises(ValueError):
        bo.ConstraintModel(None, 0.0, 1.0).eval(x=1)


def test_shard_and_merge_selection(bo):
    from bayesianoptimization_b200.sharding import merge_selection, shard_range

    assert [shard_range(10, r, 4) for r in range(4)] == [(0, 3), (3, 6), (6, 8), (8, 10)]
    rs = np.random.RandomState(0)
    for trial in range(20):
        m, world, k = 1000, 4, 7
        ys = rs.randn(m)
        ys[rs.randint(0, m, 30)] = ys[rs.randint(0, m, 30)]  # ties
        if trial % 3 == 0:
            ys[rs.randint(0, m, 5)] = np.nan
        vals = np.full((world, k + 1), np.nan)
        idxs = np.full((world, k + 1), -1, dtype=np.int64)
        for r in range(world):
            s, e = shard_range(m, r, world)
            loc = ys[s:e]
            vals[r, 0], idxs[r, 0] = loc[np.argmin(loc)], s + int(np.argmin(loc))
            order = np.argsort(loc, kind="stable")[:k]
            vals[r, 1:1 + len(order)], idxs[r, 1:1 + len(order)] = loc[order], s + order
        bi, bv, top = merge_selection(vals, idxs, k)
        assert bi == int(np.argmin(ys))
        assert list(top) == list(np.argsort(ys, kind="stable")[:k])


@pytest.mark.parametrize("driver", ["batched", "threads"])
def test_lockstep_lbfgsb_equals_sequential_runs(bo, monkeypatch, driver):
    """The n_smart L-BFGS-B runs advanced in lockstep (one batched objective call per round) follow
    exactly the iterates of independent sequential runs (R/bayes_opt/acquisition.py:365-366) - with the
    single-thread driver around SciPy's compiled core (default) and with the thread-per-run driver."""
    monkeypatch.setenv("B200BO_LBFGSB_DRIVER", driver)
    from scipy.optimize import minimize

    from bayesianoptimization_b200.fused import lockstep_lbfgsb as _lockstep_lbfgsb

    calls = []

    def acq(x):
        x = np.atleast_2d(x)
        calls.append(len(x))
        return ((x - 0.3) ** 2).sum(1) + 0.3 * np.sin(5 * x).sum(1)

    b = np.array([[0.0, 1.0]] * 4)
    seeds = np.random.RandomState(0).rand(7, 4)
    seq = [minimize(acq, s, bounds=b, method="L-BFGS-B") for s in seeds]
    n_seq = len(calls)
    calls.clear()
    lock = _lockstep_lbfgsb(acq, seeds, b)
    assert len(calls) < n_seq / 5
    for a, c in zip(seq, lock):
        assert np.array_equal(a.x, c.x) and a.fun == c.fun and a.nit == c.nit and a.success == c.success
        assert a.nfev == c.nfev and a.status == c.status and a.message == c.message and np.array_equal(a.jac, c.jac)
    # seeds on the bounds, and an objective that turns NaN (runs that fail must fail the same way)
    edge = np.vstack([np.zeros(4), np.ones(4), seeds[:2]])
    for a, c in zip([minimize(acq, s, bounds=b, method="L-BFGS-B") for s in edge], _lockstep_lbfgsb(acq, edge, b)):
        assert np.array_equal(a.x, c.x) and a.fun == c.fun and a.nit == c.nit

    def nanny(x):
        x = np.atleast_2d(x)
        return np.where(x[:, 0] > 0.5, np.nan, (x ** 2).sum(1))

    for a, c in zip([minimize(nanny, s, bounds=b, method="L-BFGS-B") for s in seeds], _lockstep_lbfgsb(nanny, seeds, b)):
        assert a.success == c.success and a.nit == c.nit and a.message == c.message
        assert np.array_equal(a.x, c.x, equal_nan=True)

    def bad(x):
        raise RuntimeError("boom")

    with pytest.raises(RuntimeError, match="boom"):
        _lockstep_lbfgsb(bad, seeds, b)
    assert len(_lockstep_lbfgsb(acq, seeds[:1], b)) == 1


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` runs without a GPU and prints ONE JSON line with the contract keys."""
    import json
    import subprocess

    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    j = json.loads(lines[0])
    if "unavailable" in j:  # no vendored reference in this checkout: the arm says so in one line and exits 0
        assert j["impl"] == "reference" and "vendor_ref" in j["unavailable"]
        pytest.skip("reference package not vendored here")
    for key in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
                "vs_baseline", "dtype", "data", "config", "impl", "cpu_baseline", "e2e"):
        assert key in j, key
    assert j["impl"] == "reference" and j["value"] > 0 and j["cpu_baseline"]["kind"] == "reference"
    assert j["e2e"]["h2d_bytes_per_step"] == 0 and "workload" in j["config"]


def test_potrf_block_emulation(tmp_path):
    """The diagonal-block Cholesky kernel's phases (csrc/potrf_block.cuh) are host/device functions;
    tools/potrf_emul.cpp runs them sequentially on the CPU: factor bit-identical to the unblocked
    algorithm, no intra-phase ordering hazards, inverse at round-off, LAPACK-style pivot index."""
    import shutil
    import subprocess

    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    exe = str(tmp_path / "potrf_emul")
    subprocess.run([gxx, "-O2", "-std=c++17", "-ffp-contract=off", "-o", exe,
                    os.path.join(ROOT, "tools", "potrf_emul.cpp")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout
    assert out.stdout.count(" ok") == 6


def test_concurrent_restart_queue_order_and_errors():
    """gpr._run_restarts_concurrently: results are stored by start index whatever thread ran them, and
    the first exception of a worker is re-raised in the caller (no GPU: fake handles, fake optimiser)."""
    import threading
    import time

    from bayesianoptimization_b200.gpr import B200GaussianProcessRegressor

    class FakeHandle:
        ptr = None

    gp = B200GaussianProcessRegressor.__new__(B200GaussianProcessRegressor)
    seen = []

    def fake_opt(obj, theta0, bounds):
        time.sleep(0.002 * (5 - theta0[0]))  # later starts finish first
        seen.append(threading.get_ident())
        return np.array([theta0[0] * 2.0]), obj(theta0)

    gp._constrained_optimization = fake_opt
    starts = [np.array([float(i)]) for i in range(5)]
    res = gp._run_restarts_concurrently([FakeHandle(), FakeHandle(), FakeHandle()], lambda h: (lambda t: -t[0]),
                                        starts, None)
    assert [r[0][0] for r in res] == [0.0, 2.0, 4.0, 6.0, 8.0]
    assert [r[1] for r in res] == [-0.0, -1.0, -2.0, -3.0, -4.0]
    assert len(set(seen)) > 1

    def failing(obj, theta0, bounds):
        if theta0[0] == 1.0:
            raise np.linalg.LinAlgError("boom")
        return theta0, 0.0

    gp._constrained_optimization = failing
    with pytest.raises(np.linalg.LinAlgError):
        gp._run_restarts_concurrently([FakeHandle(), FakeHandle()], lambda h: (lambda t: 0.0), starts, None)

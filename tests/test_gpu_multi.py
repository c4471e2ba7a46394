"""Multi-GPU (SURVEY.md 8e): the same (argmin, top-k) for any number of GPUs.

  * one process, several devices: B200GaussianProcessRegressor(devices=[...]) -> b200bo_gp_replicate +
    b200bo_multi_gpu_* (rows sharded, ONE ncclAllGather of the per-device records, merge kernel)
  * one process per GPU: torch.distributed NCCL ranks, each evaluating its contiguous shard through the
    device entry point, all_gather of the records, host merge (what bench.py does)

Both must be bit-identical to a single-GPU evaluation of the union (fp64 and fp32 mode).  Skipped on a
1-GPU machine; run on a machine with 2, 4 or 8 GPUs."""
import os
import socket
import warnings

import numpy as np
import pytest
from sklearn.gaussian_process.kernels import Matern

pytestmark = pytest.mark.gpu


def _ngpu():
    try:
        import torch

        return torch.cuda.device_count()
    except Exception:
        return 0


need2 = pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")


@pytest.fixture(scope="module")
def bo():
    import bayesianoptimization_b200 as bo

    return bo


def _synth(n, d, seed=0):
    rs = np.random.RandomState(seed)
    X = rs.uniform(size=(n, d))
    y = np.sin(X.sum(1)) + 0.1 * rs.randn(n)
    return X, y


def _fused(bo, X, y, devices=None, precision="fp64", kind="ei"):
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                         optimizer=None, devices=devices, precision=precision).fit(X, y)
    if kind == "ei":
        return bo.FusedAcquisition(bo._lib.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
    return bo.FusedAcquisition(bo._lib.ACQ_UCB, gp, kappa=2.576)


@need2
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_single_process_devices_equal_one_device(bo, precision):
    G = min(_ngpu(), 8)
    X, y = _synth(700, 6, 1)
    xt = np.random.RandomState(2).uniform(size=(60_001, 6))
    xt[59_999] = xt[5]  # a tie that straddles two shards
    f1 = _fused(bo, X, y, None, precision)
    one = f1.argmin_topk(xt, 10)
    ys = f1(xt)
    for g in sorted({2, G}):
        fg = _fused(bo, X, y, list(range(g)), precision)
        assert fg.devices == list(range(g))
        got = fg.argmin_topk(xt, 10)
        assert got[0] == one[0] and got[1] == one[1] and list(got[2]) == list(one[2]), (g, got, one)
        assert np.array_equal(fg(xt), ys)                       # even split
        # ragged split incl. an empty shard, as the L-BFGS-B driver issues it (seed r's rows on device r mod G): inside
        # an optimiser run the kernel choice is a function of the model only (PATH_STABLE), so a row's value does not
        # depend on the shard - or the device - it lands in
        xs = xt[:333]
        off = np.array([0, 10, 10] + [len(xs)] * (g - 2))[: g + 1]
        off[-1] = len(xs)
        with f1.refine_mode(), fg.refine_mode():
            assert np.array_equal(fg(xs, shard_offsets=off), f1(xs))
            assert np.array_equal(fg(xs), f1(xs))
        tiny = fg.argmin_topk(xt[:1], 3)                        # fewer rows than devices
        assert tiny[0] == 0 and list(tiny[2]) == [0]
        # throughput mode: rows depend on (seed, global index) only
        b = np.column_stack([np.zeros(6), np.ones(6)])
        p1 = f1.argmin_topk_philox(9, b, 50_000, 5)
        pg = fg.argmin_topk_philox(9, b, 50_000, 5)
        assert p1[0] == pg[0] and p1[1] == pg[1] and list(p1[3]) == list(pg[3])
        assert np.array_equal(p1[2], pg[2]) and np.array_equal(p1[4], pg[4])


@need2
def test_constrained_multi_device_and_replica_guards(bo):
    from bayesianoptimization_b200 import _lib as B

    X, y = _synth(300, 3, 4)
    c = np.cos(X.sum(1))
    xt = np.random.RandomState(3).uniform(size=(5000, 3))

    class CM:  # duck type of bayes_opt ConstraintModel as FusedAcquisition reads it
        def __init__(self, devices):
            self.model = [bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.6), alpha=1e-6,
                                                          normalize_y=True, optimizer=None, devices=devices).fit(X, c)]
            self.lb, self.ub = np.array([-0.5]), np.array([0.7])

    outs = []
    for devs in (None, [0, 1]):
        gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                             optimizer=None, devices=devs).fit(X, y)
        f = bo.FusedAcquisition(B.ACQ_POI, gp, CM(devs), xi=0.01, y_max=float(y.max()))
        outs.append((f.argmin_topk(xt, 6), f(xt)))
    assert outs[0][0][0] == outs[1][0][0] and list(outs[0][0][2]) == list(outs[1][0][2])
    assert np.array_equal(outs[0][1], outs[1][1])
    # a replica is predict-only
    hs = gp._device_handles()
    assert len(hs) == 2
    info = __import__("ctypes").c_int64()
    x_new = np.zeros(3)
    assert B.lib().b200bo_gp_append(hs[1].ptr, B.as_dp(x_new), 0.0, None) == B.ERR_STATE
    out = np.empty(4)
    assert B.lib().b200bo_gp_get(hs[1].ptr, B.GET_L, B.as_dp(out), 4) == B.ERR_STATE


@need2
def test_enabled_optimizer_with_devices_gives_the_same_suggestions(ref, bo):
    """enable(optimizer, devices=[0, 1]): the random batch is sharded and the L-BFGS-B seeds are distributed
    (seed r -> device r mod G); every value is independent of the device that produced it, so suggest() is
    bit-identical to the single-device run."""
    def f(x, y):
        return -(x**2) - (y - 1) ** 2 + 1

    outs = []
    for devs in (None, [0, 1]):
        opt = ref.BayesianOptimization(f=f, pbounds={"x": (2, 4), "y": (-3, 3)}, random_state=1, verbose=0)
        bo.enable(opt, devices=devs)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            opt.maximize(init_points=4, n_iter=0)
            sug = []
            for _ in range(3):
                s = opt.suggest()
                sug.append([s["x"], s["y"]])
                opt.register(params=s, target=f(**s))
        outs.append(np.array(sug))
    assert np.array_equal(outs[0], outs[1])


# ---------------------------------------------------------------------------------------------------
# one process per GPU (NCCL ranks), as bench.py runs
# ---------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _rank_main(rank, world, port, precision, q):
    import ctypes as C

    import torch
    import torch.distributed as dist

    import bayesianoptimization_b200 as bo
    from bayesianoptimization_b200 import _lib as B
    from bayesianoptimization_b200.sharding import merge_selection, shard_range

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    X, y = _synth(600, 5, 9)
    m, k = 100_003, 10
    xt = np.random.RandomState(21).uniform(size=(m, 5))
    xt[m - 2] = xt[11]
    gp = bo.B200GaussianProcessRegressor(kernel=Matern(nu=2.5, length_scale=0.7), alpha=1e-6, normalize_y=True,
                                         optimizer=None, device=rank, precision=precision).fit(X, y)
    f = bo.FusedAcquisition(B.ACQ_EI, gp, xi=0.01, y_max=float(y.max()))
    s0, s1 = shard_range(m, rank, world)
    shard = torch.from_numpy(xt[s0:s1]).to(dev)
    sel = torch.zeros((k + 1, 2), dtype=torch.int64, device=dev)
    B.check(B.lib().b200bo_acq_eval_dev(C.byref(f.spec), shard.data_ptr(), s1 - s0, None, None, None, k, sel.data_ptr(),
                                        s0, torch.cuda.current_stream().cuda_stream))
    gathered = torch.zeros((world, k + 1, 2), dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(gathered, sel)
    allr = gathered.cpu().numpy()
    bi, bv, top = merge_selection(allr.view(np.float64)[:, :, 0], allr[:, :, 1], k)
    if rank == 0:
        one = f.argmin_topk(xt, k)  # the union on ONE GPU
        q.put((int(bi), float(bv), [int(t) for t in top], int(one[0]), float(one[1]), [int(t) for t in one[2]]))
    dist.barrier()
    dist.destroy_process_group()


@need2
@pytest.mark.parametrize("precision", ["fp64", "fp32"])
def test_nccl_ranks_merge_equals_single_gpu_union(precision):
    import torch.multiprocessing as mp

    for world in [w for w in (2, 4, 8) if w <= _ngpu()]:
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_rank_main, args=(r, world, port, precision, q)) for r in range(world)]
        for p in procs:
            p.start()
        bi, bv, top, oi, ov, otop = q.get(timeout=300)
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
        assert bi == oi and bv == ov and top == otop, (world, precision)

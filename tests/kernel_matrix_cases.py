"""Case tables and problem builders of the covariance-variant matrix (tests/test_gpu_kernel_matrix.py).

Kept apart from the GPU test module so that the CPU-only checks (tests/test_kernel_matrix_cpu.py) can read the tables
on a machine without a device: every case kernel parses to the expected engine spec, and the tables keep covering
every covariance code on every code path of the device kernels.

Covariance codes of the device kernels (csrc/common.cuh): 0 = Matern 1/2, 1 = Matern 3/2, 2 = Matern 5/2,
3 = RBF or Matern nu=inf.
"""
import numpy as np
from sklearn.gaussian_process.kernels import RBF, ConstantKernel, Matern, WhiteKernel

NU = {"m05": 0.5, "m15": 1.5, "m25": 2.5, "minf": np.inf, "rbf": np.inf}
COV_CODE = {"m05": 0, "m15": 1, "m25": 2, "minf": 3, "rbf": 3}
DREG_MAX_D = 16  # predict: candidate coordinates stay in registers up to d = 16 (kPredictMaxDimRegs)
TILE_MAX_D = 16  # LML gradient: lml_grad_tile_kernel up to d = 16 (LG_DMAX), lml_grad_kernel above


def dreg_class(d):
    """Which phase-A instantiation of the predict kernels a dimension takes."""
    if d > DREG_MAX_D:
        return "none"
    return "even" if d % 2 == 0 else "odd"


def grad_class(d):
    return "tile" if d <= TILE_MAX_D else "generic"


# ---------------------------------------------------------------------------------------------------------------
# A. predict + acquisition.  bar: max over the five fp64 variants of the mu metric |dmu| / (|mu| + s_y) and the
# variance metric |d sigma^2| / (prior s_y^2); bar_acq: the same maximum of |d acq| / (|acq| + 1e-3) over UCB, EI and
# PoI (larger than the mu error: at training inputs sigma is a residue whose error enters the acquisition through
# z = a / sigma); bar32: the variance metric of the fp32 mode.  Every bar of this module
# is pinned at about 10x the error measured on an H100 80GB HBM3 at a 700 W power limit, and never below 1e-13 (about
# 500 ulp: below that the reference's own BLAS summation order is what varies).
# Comments: measured mu, var, acq | fp32 var.
# ---------------------------------------------------------------------------------------------------------------
PREDICT = {
    "p1": dict(kern="m05", n=1500, d=3, bar=5e-13, bar32=3e-4,
               bar_acq=1.3e-9),  # 4.8e-14 6.9e-15 1.3e-10 | 2.7e-5
    "p2": dict(kern="m05", ard=True, const=2.5, white=1e-2, n=700, d=17, bar=1e-13, bar32=4e-5,
               bar_acq=5e-12),  # 5.4e-15 4.6e-15 4.3e-13 | 3.7e-6
    "p3": dict(kern="m15", ard=True, rnd=1, n=1500, d=16, bar=2e-13, bar32=1.2e-4,
               bar_acq=2e-10),  # 1.7e-14 5.6e-15 1.8e-11 | 1.2e-5
    "p4": dict(kern="m15", const=0.3, white=1e-3, n=300, d=40, bar=1e-13, bar32=4e-5,
               bar_acq=4e-11),  # 6.9e-15 2.9e-15 3.3e-12 | 3.6e-6
    "p5": dict(kern="m25", ard=True, const=1.7, rnd=2, n=1024, d=15, bar=2e-13, bar32=8e-5,
               bar_acq=7e-9),  # 1.3e-14 3.7e-15 6.2e-10 | 8.0e-6
    "p6": dict(kern="m25", white=5e-2, n=129, d=64, bar=1e-13, bar32=1.3e-5,
               bar_acq=2e-12),  # 5.3e-15 1.4e-15 1.5e-13 | 1.3e-6
    "p7": dict(kern="rbf", const=0.5, n=1500, d=16, bar=8e-12, bar32=5e-4,
               bar_acq=3e-9),  # 7.7e-13 1.1e-14 2.7e-10 | 4.6e-5
    "p8": dict(kern="rbf", ard=True, white=1e-2, rnd=1, n=700, d=33, bar=1e-13, bar32=6e-5,
               bar_acq=3e-12),  # 4.3e-15 1.9e-15 2.7e-13 | 5.3e-6
    "p9": dict(kern="minf", n=400, d=8, bar=5e-11, bar32=2e-4,
               bar_acq=1.1e-8),  # 4.9e-12 3.4e-14 1.1e-9 | 1.8e-5
    # the remaining (code, register class) cells
    "p10": dict(kern="m05", ard=True, white=1e-3, n=257, d=2, bar=3e-13, bar32=5e-5,
                bar_acq=2e-11),  # 2.4e-14 4.4e-15 1.8e-12 | 4.8e-6
    "p11": dict(kern="m15", const=1.9, n=900, d=5, bar=3e-12, bar32=3e-4,
                bar_acq=3e-9),  # 2.5e-13 1.1e-14 2.2e-10 | 3.1e-5
    "p12": dict(kern="m25", ard=True, white=1e-2, n=2000, d=10, bar=5e-13, bar32=3.3e-4,
                bar_acq=1e-10),  # 4.4e-14 5.7e-15 1.0e-11 | 3.3e-5
    "p13": dict(kern="rbf", ard=True, const=0.8, rnd=1, n=640, d=7, bar=7e-12, bar32=2e-4,
                bar_acq=1e-9),  # 6.2e-13 9.4e-15 9.3e-11 | 1.7e-5
}

# ---------------------------------------------------------------------------------------------------------------
# B. one fused launch over a target and three constraint GPs of different covariances.  bar: max |d acq| / (|acq| +
# 1e-3) over EI and PoI (measured in the comments), pinned like A.
# ---------------------------------------------------------------------------------------------------------------
CONSTRAINED_TARGET = dict(kern="m25", ard=True)
CONSTRAINTS = [  # (kernel spec, lb, ub)
    (dict(kern="rbf", const=1.4), -0.6, 0.8),
    (dict(kern="m05", ard=True, white=1e-2), -0.9, 0.7),
    (dict(kern="m15"), -np.inf, 0.5),
]
CONSTRAINED = {
    "b17": dict(n=600, d=17, bar=2e-12),  # ei 1.6e-13 poi 2.0e-13
    "b6": dict(n=500, d=6, bar=2e-10),  # ei 4.4e-12 poi 1.6e-11
}

# ---------------------------------------------------------------------------------------------------------------
# C. fit state, LML and gradient.  Free hyper-parameters enter theta; fixed ones do not.  bar: the larger of the LML
# error |dlml| / |lml| and the gradient error max |dg| / max(|g|, 1), pinned like A.  Comments: measured lml, grad.
# ---------------------------------------------------------------------------------------------------------------
GRADIENT = {
    "g_m05_iso_tile": dict(kern="m05", n=63, d=5, const=1.3, bar=1e-13),  # 0 1.7e-15
    "g_m05_ard_tile": dict(kern="m05", ard=True, n=64, d=12, white=1e-2, bar=1e-13),  # 1.8e-16 3.8e-15
    "g_m05_iso_gen": dict(kern="m05", n=65, d=24, const=0.7, bar=1e-13),  # 0 1.9e-15
    "g_m05_ard_gen": dict(kern="m05", ard=True, n=200, d=40, bar=1e-13),  # 0 8.2e-15
    "g_m15_iso_tile": dict(kern="m15", n=700, d=16, const=2.0, const_fixed=True, bar=1e-13),  # 4.6e-16 1.8e-15
    "g_m15_ard_tile": dict(kern="m15", ard=True, n=63, d=9, const=0.8, rnd=1, bar=1e-13),  # 0 3.5e-15
    "g_m15_iso_gen": dict(kern="m15", n=64, d=17, white=5e-2, bar=1e-13),  # 1.9e-16 1.4e-15
    "g_m15_ard_gen": dict(kern="m15", ard=True, n=65, d=33, const=1.6, bar=1e-13),  # 1.6e-16 8.7e-16
    "g_m25_iso_tile": dict(kern="m25", n=200, d=3, const=1.1, ls_fixed=True, bar=6e-11),  # 5.8e-12 4.4e-12
    "g_m25_ard_tile": dict(kern="m25", ard=True, n=700, d=16, white=1e-3, white_fixed=True, bar=3e-13),  # 0 2.5e-14
    "g_m25_iso_gen": dict(kern="m25", n=63, d=64, white=2e-2, bar=1e-13),  # 1.7e-16 8.2e-15
    "g_m25_ard_gen": dict(kern="m25", ard=True, n=64, d=64, const=0.9, bar=1e-13),  # 1.6e-16 1.7e-15
    "g_rbf_iso_tile": dict(kern="rbf", n=65, d=8, bar=2e-13),  # 2.1e-15 2.0e-14
    "g_rbf_ard_tile": dict(kern="rbf", ard=True, n=200, d=6, const=1.2, rnd=2, bar=2e-13),  # 1.8e-15 1.4e-14
    "g_rbf_iso_gen": dict(kern="rbf", n=700, d=20, const=0.6, bar=4e-13),  # 1.1e-14 3.7e-14
    "g_rbf_ard_gen": dict(kern="rbf", ard=True, n=63, d=48, white=1e-2, bar=1e-13),  # 1.7e-16 3.3e-15
}

# ---------------------------------------------------------------------------------------------------------------
# D. fit() with restarts at d > 16 (lml_grad_kernel inside L-BFGS-B)
# ---------------------------------------------------------------------------------------------------------------
FIT = {
    "f_m25_iso_d32": dict(kern="m25", n=400, d=32, restarts=2, compare_theta=True),
    "f_crbf_ard_d20": dict(kern="rbf", ard=True, const=1.0, n=250, d=20, restarts=1, compare_theta=False),
}

# ---------------------------------------------------------------------------------------------------------------
# E. predict(return_cov=True) on cases of A (held to their bar), and the incremental fit (one factor row per appended
# point).  bar: the mu and variance metrics of A over all sizes, pinned like A; measured in the comments.
# ---------------------------------------------------------------------------------------------------------------
RETURN_COV = ("p1", "p3", "p6", "p8")
RETURN_COV_M = 257
APPEND = {
    "a_m05": dict(kern="m05", ard=True, const=1.8, white=2e-2, d=4, bar=1e-13),  # 1.3e-15
    "a_m15": dict(kern="m15", rnd=1, d=3, bar=2e-11),  # 1.2e-12
    "a_m25": dict(kern="m25", d=5, bar=2e-13),  # 1.4e-14
    "a_rbf": dict(kern="rbf", ard=True, const=0.6, white=5e-3, d=6, bar=1e-13),  # 5.9e-15
}
APPEND_BASE = 120
APPEND_SIZES = (121, 124, 127, 128)


# ---------------------------------------------------------------------------------------------------------------
# builders
# ---------------------------------------------------------------------------------------------------------------
def length_scale(case, d):
    """ARD: geometric spread so that no dimension is negligible; iso: about one box diagonal per sqrt(d) / 3."""
    if case.get("ard"):
        return np.geomspace(0.3, 3.0, d) * np.sqrt(d) / 4
    return 0.3 * np.sqrt(d)


def round_transform(d, rnd):
    """The kernel input transform of a space whose last ``rnd`` parameters are ints (np.round on those columns)."""
    cols = list(range(d - rnd, d))

    def transform(v):
        v = np.atleast_2d(np.asarray(v, dtype=float)).copy()
        v[:, cols] = np.round(v[:, cols])
        return v

    return transform


def base_kernel(case, d):
    """The sklearn kernel of a case, before any input transform."""
    ls = length_scale(case, d)
    lsb = "fixed" if case.get("ls_fixed") else (1e-3, 1e3)
    kern = case["kern"]
    k = RBF(ls, length_scale_bounds=lsb) if kern == "rbf" else Matern(ls, length_scale_bounds=lsb, nu=NU[kern])
    if case.get("const") is not None:
        k = ConstantKernel(case["const"], constant_value_bounds="fixed" if case.get("const_fixed") else (1e-3, 1e3)) * k
    if case.get("white") is not None:
        k = k + WhiteKernel(case["white"], noise_level_bounds="fixed" if case.get("white_fixed") else (1e-6, 1e1))
    return k


def kernel(case, d):
    """The case kernel as a user hands it to the GP: wrapped by bayes_opt's wrap_kernel when it has int columns."""
    k = base_kernel(case, d)
    if case.get("rnd"):
        from bayes_opt.parameter import wrap_kernel

        k = wrap_kernel(k, round_transform(d, case["rnd"]))
    return k


def inputs(case, n, d, rs):
    """n rows in the box: [0, 1] for float columns, [-0.5, 4.5] for the int columns (rounded by the kernel)."""
    X = rs.uniform(size=(n, d))
    r = case.get("rnd", 0)
    if r:
        X[:, d - r:] = rs.uniform(-0.5, 4.5, size=(n, r))
    return X


def problem(case, n, d, seed):
    rs = np.random.RandomState(seed)
    X = inputs(case, n, d, rs)
    y = np.sin(3 * X.sum(1) / np.sqrt(d)) + 0.5 * np.cos(2 * X[:, 0]) + 0.05 * rs.randn(n)
    return X, y, rs


def expected_spec(case):
    """(cov code, const, noise, const free, length scale free, noise free) that gpr.parse_kernel must produce."""
    has_c, has_w = case.get("const") is not None, case.get("white") is not None
    return (COV_CODE[case["kern"]], case["const"] if has_c else 1.0, case["white"] if has_w else 0.0,
            has_c and not case.get("const_fixed", False), not case.get("ls_fixed", False),
            has_w and not case.get("white_fixed", False))

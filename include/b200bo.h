/*
 * b200bo.h - C ABI of the H100-native GP-surrogate + acquisition engine.
 *
 * This is the drop-in boundary for ONE hot path of bayesian-optimization/BayesianOptimization
 * (v3.3.0): GP fit at given hyper-parameters -> batched posterior predict -> acquisition ->
 * argmin/top-k.  The reference has no FFI; its plugin surface is Python duck-typing on
 * sklearn's GaussianProcessRegressor and bayes_opt.acquisition.AcquisitionFunction
 * (SURVEY.md section 8b).  Every entry point below names the reference code it replaces
 * (R/ = R/, SK/ = site-packages/sklearn/).  INTEGRATION.md shows the ctypes
 * binding a maintainer of the reference would add.
 *
 * Conventions
 *  - plain pointers and sizes only; all matrices are row-major (C order) IEEE fp64, exactly
 *    the numpy arrays the reference passes around.
 *  - "host" entry points take HOST buffers and do their own H2D/D2H copies (synchronous).
 *    "_dev" entry points take DEVICE pointers and a cudaStream_t (as void*) and are
 *    asynchronous w.r.t. the host unless stated.
 *  - every function returns B200BO_OK (0) or a negative error code; b200bo_last_error()
 *    returns a thread-local message.  There is NO CPU fallback anywhere behind this ABI:
 *    without a CUDA device every compute entry point returns B200BO_ERR_CUDA.
 */
#ifndef B200BO_H
#define B200BO_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200BO_VERSION 200 /* 0.2.0 */

/* error codes */
#define B200BO_OK 0
#define B200BO_ERR_CUDA (-1)       /* CUDA runtime failure / no device */
#define B200BO_ERR_ARG (-2)        /* invalid argument */
#define B200BO_ERR_NOT_PD (-3)     /* kernel matrix not positive definite (np.linalg.LinAlgError) */
#define B200BO_ERR_UNSUPPORTED (-4)/* kernel / option outside the supported set (NotImplementedError) */
#define B200BO_ERR_STATE (-5)      /* handle not fitted */

/* kernel families: SK/gaussian_process/kernels.py Matern (:1685-1786), RBF (:1530-1587) */
#define B200BO_KERNEL_MATERN 0
#define B200BO_KERNEL_RBF 1
/* Matern smoothness codes */
#define B200BO_NU_05 0
#define B200BO_NU_15 1
#define B200BO_NU_25 2
#define B200BO_NU_INF 3

/* acquisition kinds: R/bayes_opt/acquisition.py:485 (UCB), :847-849 (EI), :660-661 (PoI) */
#define B200BO_ACQ_UCB 0
#define B200BO_ACQ_EI 1
#define B200BO_ACQ_POI 2
#define B200BO_ACQ_NONE 3 /* predict only: no acquisition epilogue */
/* Max-value entropy search (Wang & Jegelka, "Max-value Entropy Search for Efficient Bayesian Optimization",
 * ICML 2017).  No counterpart in the reference.  With mu, sigma the target GP's posterior (data units, as for EI)
 * and y*_0 .. y*_{K-1} the samples of the maximum set on gps[0] by b200bo_gp_set_max_values:
 *   g_k   = (y*_k - mu) / sigma
 *   alpha = (1/K) sum_{k=0..K-1}, in k order, [ g_k psi(g_k) / (2 Psi(g_k)) - log Psi(g_k) ]   (psi, Psi: N(0,1) pdf, cdf)
 *   acq_neg = -alpha [* prod_j p_j]  (the constraint factors of EI / PoI)
 * sigma = 0 (a clamped variance): alpha = 0 - the predictive distribution is a point mass.  log Psi and psi / Psi are
 * evaluated through erfcx below g = 0 and through ndtr / log1p at and above it: finite for every finite g.
 * Without a feasible registered point the constrained form still ranks candidates (EI / PoI raise there). */
#define B200BO_ACQ_MES 4
/* Log expected improvement and log probability of improvement (Ament et al., "Unexpected Improvements to Expected
 * Improvement for Bayesian Optimization", NeurIPS 2023).  No counterpart in the reference.  With mu, sigma,
 * a = mu - y_max - xi and z = a / sigma exactly as for EI / PoI, and h(z) = phi(z) + z Phi(z):
 *   LOGEI:  alpha = log h(z) + log sigma       (= log EI)
 *   LOGPOI: alpha = log Phi(z)                 (= log PoI)
 *   acq_neg = -(alpha + sum_j log p_j)          (the constraint factors in log space, summed in j order)
 * log h takes three branches: log(phi + z Phi) above z = -1; below it log phi(z) + log(1 - sqrt(pi/2) |z| erfcx(-z/sqrt2))
 * through log1mexp; below z = -2^26 the asymptote -z^2/2 - log(2 pi)/2 - 2 log|z|.  log Phi and log p_j go through
 * erfcx in the lower tail (a pair of bounds in one tail is reflected so that both arguments are <= 0), so both are
 * finite where EI, PoI or p_j underflow to 0.  sigma = 0: alpha = log of the EI / PoI limit (-inf for a < 0, NaN for
 * a = 0); a constraint GP with sigma = 0 makes the value NaN, as for EI / PoI. */
#define B200BO_ACQ_LOGEI 6
#define B200BO_ACQ_LOGPOI 7
/* Code 5 is not assigned: it is rejected as an unknown kind (B200BO_ERR_ARG), as before these kinds existed. */
/* Noisy expected improvement and its log (Letham, Karrer, Ottoni & Bakshy, "Constrained Bayesian Optimization with
 * Noisy Experiments", Bayesian Analysis 2019; Ament et al. 2023 for the log form).  No counterpart in the reference.
 * gps[0] is the NOISELESS handle holding S fantasies (b200bo_gp_set_fantasies): A = K0^-1 F and best_0 .. best_{S-1}.
 * With k* = const_value k(xs, Xs), mu_s = y_std k*^T a_s + y_mean, sigma0 the noiseless GP's posterior sd (data
 * units, the negative-variance clamp counted as usual) and a_s = mu_s - best_s - xi:
 *   NEI:    alpha = (1/S) sum_{s=0..S-1}, in s order, EI(a_s, sigma0)                 (EI's formula and sigma = 0 rules)
 *   LOGNEI: alpha = M + log sum_s exp(l_s - M) - log S,  l_s = LogEI(a_s, sigma0),  M = max_s l_s
 *           (-inf when every l_s is -inf; NaN when any l_s is NaN)
 *   acq_neg = -alpha * prod_j p_j  (NEI)   or   -(alpha + sum_j log p_j)  (LOGNEI), the constraint GPs as for EI / LogEI.
 * Served by the 16-warp fp64 kernel on its bulk-copy phase-B pipes (the default and the multicast one; host / device /
 * Philox candidates), the small-batch kernels and b200bo_acq_value_grad, in fp64 whatever the handle's precision.  The
 * 8-warp, DFMA and fp32 kernels and the cp.async / m8n8k4 phase B selected by the A/B switches return
 * B200BO_ERR_UNSUPPORTED.  Never pruned.  mu / sd outputs (d_mu, d_sd) are refused with B200BO_ERR_ARG (there is no
 * single mean).  Gradient: d NEI = (1/S) sum_s [Phi(z_s) d mu_s + phi(z_s) d sigma0]; d LogNEI = sum_s p_s d l_s with
 * p_s = exp(l_s - M) / sum exp(l - M) (LogEI's per-fantasy derivative, softmax-weighted). */
#define B200BO_ACQ_NEI 8
#define B200BO_ACQ_LOGNEI 9
/* Constrained noisy expected improvement and its log (Letham et al. 2019, with noisy constraints; DESIGN.md 4.15).
 * No counterpart in the reference.  Every GP of the call is a NOISELESS handle holding fantasies with the same S and
 * n: gps[0] the target's (b200bo_gp_set_fantasies, then usually b200bo_gp_set_fantasy_incumbent for best_s), gps[j],
 * j >= 1, constraint j's (A_j = K0_j^-1 F_j; its best_s are not used).  With mu_s and sigma0 from gps[0] as for NEI,
 * mu_js = y_std_j k_j*^T a_js + y_mean_j and sigma0_j the posterior sd of gps[j] (data units):
 *   P_js = Phi((ub_j - mu_js)/sigma0_j) - Phi((lb_j - mu_js)/sigma0_j)   (the factor rules of EI's constraints)
 *   CNEI:    alpha = (1/S) sum_{s=0..S-1}, in s order, EI(a_s, sigma0) * P_1s * .. * P_Js       (products in j order)
 *   LOGCNEI: alpha = M + log sum_s exp(l_s - M) - log S,  l_s = LogEI(a_s, sigma0) + sum_j log P_js  (log_cfactor)
 *            (-inf when every l_s is -inf; NaN when any l_s is NaN)
 *   acq_neg = -alpha.
 * Without constraint GPs (n_gps = 1) the value is NEI / LOGNEI.  Served where NEI is (the 16-warp fp64 kernel on its
 * bulk-copy pipes with host, device and Philox candidates, and the small-batch kernels); everything NEI refuses returns
 * B200BO_ERR_UNSUPPORTED.  b200bo_acq_value_grad serves both kinds (small-batch path), by the product rule per sample:
 * d CNEI = (1/S) sum_s [prod_j P_js dEI_s + EI_s sum_j (prod_{k != j} P_ks) dP_js]; d LOGCNEI = sum_s p_s d l_s with
 * p_s = exp(l_s - M) / sum exp(l - M).  Never pruned.  mu / sd outputs: B200BO_ERR_ARG.  A GP
 * without fantasies: B200BO_ERR_STATE; handles with different S or n: B200BO_ERR_ARG. */
#define B200BO_ACQ_CNEI 10
#define B200BO_ACQ_LOGCNEI 11
/* Posterior-mean merit, for recommending a point at the end of a noisy run (Letham et al. 2019 recommend the best
 * posterior mean; DESIGN.md 4.17).  No counterpart in the reference, whose TargetSpace.max() is the largest noisy
 * observation.  With mu_j the posterior mean of gps[j] (data units) and A1 = sum_i |alpha_i| of gps[0] (normalised
 * units):
 *   viol(x)  = sum_{j=1..J}, in j order, (max(0, lb_j - mu_j) + max(0, mu_j - ub_j))
 *   merit(x) = mu_0                     if viol(x) = 0
 *            = -T (1 + viol(x))         otherwise,   T = 2 B + 1,  B = |y_mean| + y_std const_value A1 >= |mu_0|
 *   acq_neg  = -merit(x)                (-mu_0 without constraint GPs)
 * so every mean-feasible candidate ranks above every infeasible one.  This is the rule: it is not a product of
 * probabilities, and it needs no sigma.  For a one-sided bound, viol_j = 0 is a marginal probability of feasibility of
 * at least 1/2.  An infinite bound contributes 0 (the short-circuits of the constraint factors); the sums, max (NaN-
 * propagating), add and multiply are evaluated without FMA contraction, as for b200bo_cpaths_eval.  Served by the
 * host, device and Philox entry points, the multi-GPU entry points and b200bo_acq_value_grad, always in fp64 and
 * never pruned: one mean-only tile kernel (no L^-1 product) or the small-batch kernels.  mu_0 of a batch served by
 * the tile kernel is bit-equal to the mean b200bo_gp_predict returns for it on an fp64 handle.  d_mu is allowed;
 * d_sd -> B200BO_ERR_ARG.  The A/B switches B200BO_PREDICT_* and B200BO_PRUNE* do not apply.  Gradient: -d mu_0 on a
 * feasible row (viol = 0), T sum_j d viol_j on an infeasible one (d viol_j = -d mu_j below lb_j, +d mu_j above ub_j). */
#define B200BO_ACQ_MEAN 12

#define B200BO_MAX_GPS 8   /* 1 target GP + up to 7 constraint GPs per call */
#define B200BO_MAX_DIM 64  /* max input dimension d */
#define B200BO_MAX_TOPK 64 /* max n_smart seeds returned by argmin_topk */

/* per-dimension input transforms of bayes_opt.parameter.wrap_kernel
 * (R/bayes_opt/parameter.py:484-487): identity for floats (:222-234), np.round for ints (:308-320) */
#define B200BO_XFORM_IDENTITY 0
#define B200BO_XFORM_ROUND 1

typedef struct b200bo_gp b200bo_gp; /* opaque: one GP's device-resident factorisation */

/* kernel hyper-parameters: const_value * k(x/length_scale, x'/length_scale) [+ noise_level * delta(x, x')]
 * (ConstantKernel * {Matern,RBF} [+ WhiteKernel]; const_value = 1 for a bare kernel, noise_level = 0 without a
 * WhiteKernel term, SK/gaussian_process/kernels.py:1205-1330: the term adds noise_level to the diagonal of K(X,X)
 * and to the prior variance kernel_.diag(X*), and nothing to K(X*,X)). */
typedef struct {
    int32_t family;            /* B200BO_KERNEL_* */
    int32_t nu;                /* B200BO_NU_* (ignored for RBF) */
    int32_t n_length_scale;    /* 1 (isotropic) or d (anisotropic) */
    int32_t reserved;
    double const_value;        /* ConstantKernel factor; 1.0 when absent */
    const double* length_scale;/* host pointer, n_length_scale entries */
    double noise_level;        /* WhiteKernel term; 0.0 when absent */
} b200bo_kernel;

/* One acquisition evaluation: the closure built by AcquisitionFunction._get_acq
 * (R/bayes_opt/acquisition.py:171-219):  -base_acq(mu, sigma) [* prod_j p_j(x)]. */
/* Which kernels evaluate a batch.  AUTO: the tiled persistent kernel or the small-batch kernels, chosen
 * from the batch size m.  STABLE: chosen from the model size only - an optimiser's objective f(x) and its
 * finite-difference stencil f(x + h e_i) arrive as batches of different sizes and must be summed in the same
 * order (SP/optimize/_numdiff.py forms (f(x+h) - f(x)) / 1.5e-8). */
#define B200BO_PATH_AUTO 0
#define B200BO_PATH_STABLE 1

typedef struct {
    int32_t kind;              /* B200BO_ACQ_* */
    int32_t n_gps;             /* 1 + number of constraint GPs */
    int32_t path;              /* B200BO_PATH_* */
    int32_t reserved;
    double kappa;              /* UCB */
    double xi;                 /* EI / PoI */
    double y_max;              /* EI / PoI */
    b200bo_gp* gps[B200BO_MAX_GPS]; /* gps[0] = target GP; gps[1..] = ConstraintModel GPs */
    double lb[B200BO_MAX_GPS]; /* lb[j], ub[j] for gps[j] (j >= 1); +-inf allowed */
    double ub[B200BO_MAX_GPS]; /* (R/bayes_opt/constraint.py:200-221) */
} b200bo_acq;

/* ---- library / device ---------------------------------------------------------------- */
int b200bo_version(void);
const char* b200bo_last_error(void);
int b200bo_device_count(void);
/* number of kernel launches issued by this library in this process so far (bench.py's
 * gpu_launches claim is the difference across the timed region). */
int64_t b200bo_launch_count(void);

/* ---- GP handle ------------------------------------------------------------------------ */
int b200bo_gp_create(b200bo_gp** out, int device);
void b200bo_gp_destroy(b200bo_gp* gp);

/* Arithmetic of the N^2 term (V = L^-1 K*^T and sum V^2) in the fused predict/acquisition kernel:
 *   B200BO_PRECISION_FP64  exact fp64 (mma.sync f64 / DFMA); parity bar 1e-5 (default)
 *   B200BO_PRECISION_FP32  "fp32 mode": 3xTF32 on wgmma tensor cores, fp32 accumulate in registers;
 *                          K*, the mean and the acquisition epilogue stay fp64; tolerance 1e-3.
 * A call uses the precision of gps[0].  (BASELINE configs[2]: fp32 vs fp64 tolerance.) */
#define B200BO_PRECISION_FP64 0
#define B200BO_PRECISION_FP32 1
int b200bo_gp_set_precision(b200bo_gp* gp, int precision);

/* enable != 0: the handle's fit-side work (set_data / fit / lml) is issued on a CUDA stream of its own
 * instead of the legacy default stream, so that several handles driven from different host threads
 * factorise concurrently - the independent L-BFGS-B restarts of the hyper-parameter search
 * (SK/gaussian_process/_gpr.py:321-340 runs them one after the other).  Every entry point still returns
 * with its results complete; handles are not thread-safe individually (one thread per handle). */
int b200bo_gp_set_private_stream(b200bo_gp* gp, int enable);

/* Optional per-dimension input transform (wrap_kernel); xform has d entries or NULL. Must be
 * set before fit.  Replaces R/bayes_opt/parameter.py:484-487 for float/int parameters. */
int b200bo_gp_set_transform(b200bo_gp* gp, const int32_t* xform, int d);

/* Samples y*_0 .. y*_{K-1} of the maximum for B200BO_ACQ_MES (data units), stored as a host copy on this handle and
 * passed to the kernel by value when the handle is gps[0] of an MES call.  0 <= K <= B200BO_MAX_PATHS; K = 0 clears
 * them.  Non-finite values or K out of range: B200BO_ERR_ARG.  An MES call whose gps[0] holds none returns
 * B200BO_ERR_STATE.  Fits keep them; a replica (b200bo_gp_replicate) is a handle of its own and needs its own call. */
int b200bo_gp_set_max_values(b200bo_gp* gp, const double* ystar, int K);

/* Fantasies for B200BO_ACQ_NEI / B200BO_ACQ_LOGNEI (DESIGN.md 4.13).  `noisy` is the fitted GP, K = const_value
 * k(Xs, Xs) + sigma_n^2 I with sigma_n^2 = alpha + noise_level; `noiseless` is b200bo_gp_fit on the same data with the
 * WhiteKernel term dropped and alpha = tau, K0 = const_value k(Xs, Xs) + tau I.  noisy may equal noiseless
 * (sigma_n^2 = tau).  z, e: (n, S) host draws, row-major; incumbent: (n,) host mask of the registered rows that may be
 * the incumbent.  In the normalised units of the fit (y_n the normalised targets, L0 = chol(K0)):
 *   F_prior = L0 Z,   R = y_n 1^T - F_prior - sqrt(sigma_n^2 - tau) E,
 *   F = y_n 1^T - sqrt(sigma_n^2 - tau) E - (sigma_n^2 - tau) K^-1 R,   A = K0^-1 F,
 *   best_s = max over incumbent rows i of (y_std F_is + y_mean).
 * Column s of F is a joint sample of the latent values at X (Matheron's rule, exact for the kernel const_value k + tau
 * delta observed with noise sigma_n^2 - tau).  The N^2 work (one product with L0, one solve with K and one with K0 per
 * sample: O(N^2 S)) runs on the device with the solve and matvec kernels of the fit.  A (np x S, zero padded) and
 * best_s behind it are stored on `noiseless` in device memory (the kernels evaluate NEI out of line from pointers).  f_out (nullable, (n, S) host) receives F in data
 * units (y_std F + y_mean), best_out (nullable, (S,) host) best_s.  1 <= S <= B200BO_MAX_PATHS.  B200BO_ERR_ARG: handles
 * on different devices, a different n, d or y statistics, noiseless with a WhiteKernel term, sigma_n^2 < tau, an empty
 * incumbent mask, non-finite draws; B200BO_ERR_STATE: a handle not fitted or a replica.  A later fit, append, condition
 * or set_transform on `noiseless` drops the fantasies; an NEI call on it then returns B200BO_ERR_STATE. */
int b200bo_gp_set_fantasies(b200bo_gp* noiseless, const b200bo_gp* noisy, const double* z, const double* e, int S,
                            const uint8_t* incumbent, double* f_out, double* best_out);

/* Per-sample incumbents for B200BO_ACQ_CNEI / B200BO_ACQ_LOGCNEI (DESIGN.md 4.15).  eligible: (n, S) host mask,
 * row-major: eligible[i*S + s] != 0 when row i may be sample s's incumbent (in the caller's rule: within the bounds
 * and feasible under sample s's constraint fantasies).  Recomputes, on the device copy and the host copy,
 *   best_s = max over eligible rows i of (y_std F_is + y_mean),
 *   or, when no row is eligible in sample s, min over all n rows of (y_std F_is + y_mean)
 * (a floor: EI against it still rewards objective value and feasibility together).  best_out (nullable, (S,) host)
 * receives best_s.  NULL handle or mask -> B200BO_ERR_ARG; not fitted, a replica, no fantasies, or fantasies
 * conditioned on pending rows -> B200BO_ERR_STATE.  A later fit, append or condition drops them with the fantasies. */
int b200bo_gp_set_fantasy_incumbent(b200bo_gp* noiseless, const uint8_t* eligible, double* best_out);

/* Per-sample incumbents of CNEI / LogCNEI formed on the device (DESIGN.md 4.16), on unconditioned handles and on
 * handles conditioned on pending rows (b200bo_gp_condition_fantasies) alike.  target: the target's noiseless handle;
 * constraints[j], j < n_constraints (0..7): constraint j's noiseless handle, all with the target's S, n (registered plus
 * pending rows), np and device.  in_bounds: (n,) host mask, nonzero when row i lies within the parameter bounds.  From
 * the F every handle keeps, in data units v = y_std F + y_mean formed without FMA contraction (so v equals the host
 * copies b200bo_gp_set_fantasies and b200bo_gp_condition_fantasies return, bit for bit), row i is eligible in sample s
 * when in_bounds[i] != 0 and lb[j] <= v_j[i, s] <= ub[j] for every j, and
 *   best_s = max over eligible rows of v_target[i, s],  or, with no eligible row, min over all n rows of v_target[i, s]
 * - b200bo_gp_set_fantasy_incumbent's rule with that mask, bit for bit.  Writes best_s behind the target's A and into
 * its host copy; best_out (nullable, (S,) host) receives it.  No fantasy matrix is copied to the host.  NULL handles,
 * in_bounds, or lb / ub with n_constraints > 0, n_constraints outside [0, 7], a different S, n, np or device, or
 * !(lb[j] < ub[j]) -> B200BO_ERR_ARG; a handle not fitted, a replica, or without fantasies -> B200BO_ERR_STATE. */
int b200bo_gp_set_constrained_incumbent(b200bo_gp* target, b200bo_gp* const* constraints, int n_constraints,
                                        const double* lb, const double* ub, const uint8_t* in_bounds,
                                        double* best_out);

/* Replaces the tail of GaussianProcessRegressor.fit (SK/gaussian_process/_gpr.py:275-285,
 * :349-367): y normalisation, K = k(X,X), K_ii += alpha, L = chol(K), alpha_ = K^-1 y, plus
 * the triangular inverse L^-1 the predict kernel streams.  X: (n,d) host, y: (n,) host.
 * Returns B200BO_ERR_NOT_PD when the factorisation meets a non-positive pivot; *info (nullable)
 * then receives the 1-based pivot index (LAPACK dpotrf convention). */
int b200bo_gp_fit(b200bo_gp* gp, const double* X, const double* y, int64_t n, int d,
                  const b200bo_kernel* kern, double alpha, int normalize_y, int64_t* info);

/* Incremental factor update (no counterpart in the reference, which always re-factorises:
 * R/bayes_opt/acquisition.py:84, :1130-1135): append ONE training point at the hyper-parameters of
 * the last b200bo_gp_fit in O(N^2) - new row of K, L (pivot checked) and L^-1, new y statistics and
 * alpha_.  Results equal a from-scratch fit on the extended data to round-off.  Returns
 * B200BO_ERR_STATE when the padded capacity is exhausted (caller refits), B200BO_ERR_NOT_PD as fit. */
int b200bo_gp_append(b200bo_gp* gp, const double* x_new, double y_new, int64_t* info);

/* ---- Kriging believer: conditioning on pending points (DESIGN.md 4.11) ----------------------
 * (Ginsbourger, Le Riche & Carraro, "Kriging is well-suited to parallelize optimization", 2010.)  No counterpart in
 * the reference, whose ConstantLiar refits the GP on dummy targets (R/bayes_opt/acquisition.py:1058-1148).
 *
 * b200bo_gp_fork: a new, full and appendable handle on src's device (not a predict-only replica) holding src's fitted
 * state - X / Xs, K, L, L^-1 and its transpose, alpha_, y, the y statistics, the transform, the hyper-parameters, the
 * precision, the MES samples and the NEI fantasies (A re-pitched, best_s, F, Z, W) - with capacity np' = ceil((n + extra_rows)/128)*128 rows.  The N^2 matrices are
 * re-pitched from np to np' with identity padding.  Extra device memory: about 4 * 8 * np'^2 bytes, plus the stage
 * images of L^-1 the predict kernels build on first use.  np' == np: predictions, acquisitions and selections are
 * bit-equal to src's; np' > np: equal to round-off.  The fork's training set is for conditioning / appending:
 * b200bo_gp_lml on it needs b200bo_gp_set_data first.  Out of memory: B200BO_ERR_CUDA; src not fitted or a replica:
 * B200BO_ERR_STATE.  n + extra_rows <= 38000. */
int b200bo_gp_fork(const b200bo_gp* src, int64_t extra_rows, b200bo_gp** out);
/* Conditions gp in place on the p rows of Xp ((p,d) host), one O(N^2) row update each, at the hyper-parameters and y
 * statistics of the last fit.  Row r's target is the believer value mu(Xp[r]) of the GP conditioned on rows 0..r-1,
 * which equals the mean of the GP before the call (alpha_ extends by zeros: K'[alpha_; 0] = [y; k^T alpha_]), so the
 * posterior mean does not change anywhere and only the variance shrinks near the rows.  mu_out (nullable, (p,) host)
 * receives the believer values in data units; they also become the rows' targets (b200bo_gp_append on the result
 * treats them as data).  Errors: not fitted or a replica, or p > np - n (no slack: fork first) -> B200BO_ERR_STATE;
 * non-finite Xp -> B200BO_ERR_ARG; a non-positive pivot -> B200BO_ERR_NOT_PD with the 1-based index of the failing
 * row in the message (LAPACK dpotrf convention), and the handle is left unfitted. */
int b200bo_gp_condition(b200bo_gp* gp, const double* Xp, int64_t p, double* mu_out);

/* ---- NEI with pending points (DESIGN.md 4.14) -------------------------------------------------
 * (Letham et al. 2019: the values at pending points are drawn jointly with the fantasies.)  `noiseless` holds S
 * fantasies (b200bo_gp_set_fantasies, or a fork of such a handle: b200bo_gp_fork carries A, best_s, F, the prior draws Z
 * and W = K^-1 R of the registered rows).  Conditions it in place on the p rows of Xp ((p,d) host) as
 * b200bo_gp_condition does (same row update, believer targets, y statistics), and per row j, with the new row
 * [l^T, r] of L0 and zp[j] (the (p,S) host array, row-major) its fresh standard-normal draws:
 *   F_js = l^T [Z_s; z_1s .. z_(j-1)s] + r z_js + const_value k(x_j, X_reg)^T W_s      (normalised units)
 * - the joint prior draw at x_j from the grown factor plus the Matheron update over the registered rows - then
 * best_s = max(best_s, y_std F_js + y_mean): pending rows always count toward the incumbent.  After the last row
 * A' = K0'^-1 F' per sample with the explicit-inverse solve and one refinement step of b200bo_gp_set_fantasies.  With
 * sigma_n^2 = tau, F_js = mu(x_j) + (the l^T z terms of the pending rows) + r z_js.  The handle is then an ordinary NEI
 * handle over X u P.  p single-row calls give bit-equal results to one p-row call; p = 0 changes nothing.  f_out
 * (nullable, (p,S) host) receives F_j. in data units, best_out (nullable, (S,) host) best_s.  Errors, in this order:
 * NULL arguments or p < 0 -> B200BO_ERR_ARG; not fitted or a replica, p > np - n (no slack: fork first), no fantasies ->
 * B200BO_ERR_STATE; non-finite Xp or zp -> B200BO_ERR_ARG; a non-positive pivot -> B200BO_ERR_NOT_PD with the 1-based
 * index of the failing row in the message, or non-finite fantasies -> B200BO_ERR_NOT_PD; after either the handle holds
 * no fantasies (and after a pivot failure it is unfitted).  b200bo_gp_condition on the handle drops the fantasies. */
int b200bo_gp_condition_fantasies(b200bo_gp* noiseless, const double* Xp, int64_t p, const double* zp, double* f_out,
                                  double* best_out);

/* Replaces GaussianProcessRegressor.log_marginal_likelihood(theta, eval_gradient)
 * (SK/gaussian_process/_gpr.py:541-656) on the training set of the last b200bo_gp_set_data /
 * b200bo_gp_fit call.  grad (nullable) receives d LML / d log(theta): [log const_value if
 * has_const & 1], then log length_scale (1 or d entries), then [log noise_level if has_const & 2].
 * Non-PD -> *lml = -inf, grad = 0 (as :590-593) and the call still returns B200BO_OK. */
int b200bo_gp_set_data(b200bo_gp* gp, const double* X, const double* y, int64_t n, int d,
                       int normalize_y);
int b200bo_gp_lml(b200bo_gp* gp, const b200bo_kernel* kern, double alpha, int has_const,
                  double* lml, double* grad);

/* Read back fitted state (tests / sklearn attribute parity: L_, alpha_, _y_train_mean/_std). */
#define B200BO_GET_L 0        /* (n,n) lower Cholesky factor, upper triangle zero */
#define B200BO_GET_ALPHA 1    /* (n,) alpha_ */
#define B200BO_GET_YSTATS 2   /* (2,) y_mean, y_std */
#define B200BO_GET_K 3        /* (n,n) K + alpha*I */
#define B200BO_GET_LINV 4     /* (n,n) L^-1 (lower) */
int b200bo_gp_get(b200bo_gp* gp, int what, double* out, int64_t len);
int64_t b200bo_gp_n(const b200bo_gp* gp);
int b200bo_gp_dim(const b200bo_gp* gp);

/* ---- predict / acquisition: HOST buffers --------------------------------------------- */
/* Replaces GaussianProcessRegressor.predict(X, return_std) (SK/gaussian_process/_gpr.py:446-500).
 * Xc: (m,d) host; mu: (m,) host; sd: (m,) host or NULL (mean only); n_clamped (nullable)
 * receives the number of negative variances set to 0 (the reference warns, :485-491). */
int b200bo_gp_predict(b200bo_gp* gp, const double* Xc, int64_t m, double* mu, double* sd,
                      int64_t* n_clamped);

/* Replaces GaussianProcessRegressor.predict(X, return_cov=True) (SK/gaussian_process/_gpr.py:464-475):
 * cov = (K(X*,X*) - V^T V) * y_std^2 with V = L^-1 K*^T.  mu: (m,), cov: (m,m) host.  1 <= m <= 16384.
 * The only caller in the reference is BayesianOptimization.predict (R/bayes_opt/bayesian_optimization.py:238). */
int b200bo_gp_predict_cov(b200bo_gp* gp, const double* Xc, int64_t m, double* mu, double* cov);

/* Replaces the closure returned by AcquisitionFunction._get_acq (R/bayes_opt/acquisition.py:
 * 171-219) incl. ConstraintModel.predict (R/bayes_opt/constraint.py:153-221):
 * acq_neg[i] = -base_acq(mu_i, sigma_i) * prod_j p_j(x_i).  Xc: (m,d) host, acq_neg: (m,) host. */
int b200bo_acq_eval(const b200bo_acq* spec, const double* Xc, int64_t m, double* acq_neg);

/* Value and analytic input gradient of the same closure: val[i] = the value b200bo_acq_eval returns for row i,
 * grad[i*d + j] = d val[i] / d x_ij, for every acquisition kind and 0 .. B200BO_MAX_GPS - 1 constraint GPs.
 * Xc: (m,d) host, val: (m,), grad: (m,d) host.  Always runs on the fp64 small-batch kernels (meant for tens to
 * hundreds of rows; a GP in fp32 precision takes the same fp64 path), on the device of the spec's GPs.  val is
 * bit-equal to b200bo_acq_eval on the small-batch path (B200BO_SMALL_PATH=1) and, like the gradient, depends on the
 * row only.  A dimension with B200BO_XFORM_ROUND has gradient 0; at a training input the Matern nu=0.5 kernel's kink
 * contributes 0; where the variance is clamped to 0, d sigma is taken as 0; a NaN value gives a NaN gradient row. */
int b200bo_acq_value_grad(const b200bo_acq* spec, const double* Xc, int64_t m, double* val, double* grad);

/* Replaces AcquisitionFunction._random_sample_minimize's evaluation + selection
 * (R/bayes_opt/acquisition.py:311-317): evaluates the closure on Xc and returns
 *   best_idx/best_val = np.argmin semantics (first NaN wins; ties -> lowest index),
 *   topk_idx/topk_val = the k smallest in (value, index) order, NaN last (np.argsort order).
 * acq_neg (nullable) additionally receives all m values.  The values are NOT materialised otherwise: every CTA of the
 * fused kernel keeps its k best (key, index) pairs and a small kernel merges the lists.  Batches of >= 2 chunks
 * (8 x 128 x #SM rows) are uploaded chunk by chunk on a copy stream behind the kernel.  A NaN / inf candidate coordinate
 * is detected where the kernels read it and reported as B200BO_ERR_ARG ("Input X contains NaN or infinity.", what
 * sklearn's validate_data raises on the reference path); the same holds for b200bo_acq_eval / b200bo_gp_predict. */
int b200bo_acq_argmin_topk(const b200bo_acq* spec, const double* Xc, int64_t m, int k,
                           double* best_val, int64_t* best_idx, double* topk_val,
                           int64_t* topk_idx, double* acq_neg);

/* ---- predict / acquisition: DEVICE buffers (candidates resident in HBM) --------------- */
/* d_Xc: (m,d) device fp64.  d_acq_neg, d_mu, d_sd: (m,) device or NULL.
 * If k > 0: d_sel receives (k+1) records {double value; int64 index}: record 0 = argmin,
 * records 1..k = top-k (device memory, 16*(k+1) bytes).  index_base is added to every index
 * (global index of this shard's first candidate).  stream: cudaStream_t. */
int b200bo_acq_eval_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m,
                        double* d_acq_neg, double* d_mu, double* d_sd, int k, void* d_sel,
                        int64_t index_base, void* stream);

/* ---- throughput mode: device-side candidate source ------------------------------------ */
/* The reference draws the M candidates on the host (TargetSpace.random_sample, R/bayes_opt/target_space.py:
 * 565-603: column j = rng.uniform(lo_j, hi_j, M) from MT19937) - ~10^8 doubles/s, slower than the fp32-mode
 * kernel consumes them.  In throughput mode candidate i, column j is  lo_j + (hi_j - lo_j) * u,  u the 53-bit
 * uniform from Philox4x32-10 with counter (i + index_base, j/2) and key `seed`, generated INSIDE the fused
 * kernel: the candidate matrix never exists in host memory or HBM.  Rows depend only on (seed, global index),
 * so results are identical for any tiling and any number of GPUs.  This is an opt-in mode: it does not
 * reproduce the reference's RNG stream (parity mode = the host entry points above).
 * lo, hi: (d,) host.  best_x: (d,), topk_x: (k,d) host - the winners' coordinates, regenerated on the device. */
int b200bo_acq_argmin_topk_philox(const b200bo_acq* spec, uint64_t seed, const double* lo, const double* hi,
                                  int64_t m, int64_t index_base, int k, double* best_val, int64_t* best_idx,
                                  double* best_x, double* topk_val, int64_t* topk_idx, double* topk_x);
/* Device-resident flavour: only the (k+1) selection records are produced (d_sel as in b200bo_acq_eval_dev). */
int b200bo_acq_select_philox_dev(const b200bo_acq* spec, uint64_t seed, const double* lo, const double* hi,
                                 int64_t m, int64_t index_base, int k, void* d_sel, void* stream);
/* Rows of the Philox candidate matrix for given global indices (idx < 0 -> NaN row).  out: (n_idx, d) host. */
int b200bo_philox_rows(int device, uint64_t seed, const double* lo, const double* hi, int d,
                       const int64_t* idx, int64_t n_idx, double* out);

/* ---- multi-GPU (one process, several devices of one box) -------------------------------- */
/* SURVEY.md 8e: candidates are independent given the model, so a batch shards by rows over G devices, the
 * O(N^2) model state is replicated, and ONE exchange merges the per-device (argmin, top-k) records:
 * an ncclAllGather of (k+1) 16-byte records per device over NVLink (communicators from ncclCommInitAll,
 * created on first use for a device list and cached), then a merge kernel on device 0.  The reference has no
 * counterpart (single process, single thread: R/bayes_opt/acquisition.py:274-320).
 *
 * b200bo_gp_replicate: copy the fitted state of `src` (what predict needs: scaled X, L^-1, alpha_, statistics)
 * to a new handle on `device` with peer copies - no re-factorisation.  The replica is predict-only. */
int b200bo_gp_replicate(const b200bo_gp* src, int device, b200bo_gp** out);
/* specs[g] is the acquisition on device g (its gps[] are handles living on ONE device; all specs describe the
 * same model).  Rows [m*g/G, m*(g+1)/G) go to device g (remainder to the low devices); results as
 * b200bo_acq_argmin_topk with GLOBAL row indices - bit-identical to the single-device call. */
int b200bo_multi_gpu_acq_argmin_topk(const b200bo_acq* specs, int n_dev, const double* Xc, int64_t m, int k,
                                     double* best_val, int64_t* best_idx, double* topk_val,
                                     int64_t* topk_idx);
int b200bo_multi_gpu_acq_argmin_topk_philox(const b200bo_acq* specs, int n_dev, uint64_t seed, const double* lo,
                                            const double* hi, int64_t m, int64_t index_base, int k,
                                            double* best_val, int64_t* best_idx, double* best_x,
                                            double* topk_val, int64_t* topk_idx, double* topk_x);
/* Closure values for a batch split over the devices: rows [offsets[g], offsets[g+1]) on device g
 * (offsets: (n_dev+1,) host, or NULL for an even split).  Used by the lockstep L-BFGS-B driver to run seed r's
 * requests on device r mod G (R/bayes_opt/acquisition.py:364-374).  No collective. */
int b200bo_multi_gpu_acq_eval(const b200bo_acq* specs, int n_dev, const double* Xc, int64_t m,
                              const int64_t* offsets, double* acq_neg);

/* ---- posterior sample paths (Thompson sampling) ------------------------------------------ */
/* The reference has no counterpart in the package; its tutorial's custom ThompsonSampling
 * (R/examples/acquisition_functions.ipynb) draws multivariate_normal(mean, cov) on the host from
 * predict(X, return_cov=True), O(M^3) in the number of candidates.  A path here is a fixed smooth function
 * (pathwise conditioning, Wilson et al. ICML 2020), in the normalised units of the fitted state:
 *   path_p(x) = y_std * ( sum_l w[l][p] phi_l(xs) + sum_i v[i][p] k(xs, Xs_i) ) + y_mean,  xs = transform(x)/ls
 *   phi_l(xs) = sqrt(2 const_value / L) cos(omega_l . xs + b_l)
 *   v = K^-1 (y_norm - Phi(Xs) w - eps)      (K incl. alpha + noise_level on the diagonal, as in fit)
 * A path samples the latent function: the WhiteKernel term enters eps and K's diagonal, not the path.
 * Every draw crosses the ABI as an array, so the caller's RNG stays the only source of randomness:
 *   omega: (L,d) unit-length-scale spectral draws (standard normal for RBF; multivariate t with 2 nu degrees of
 *          freedom for Matern nu), b: (L,) phases in [0, 2 pi), w: (L,q) N(0,1) weights, eps: (n,q) noise draws
 *          with variance alpha + noise_level.  All row-major host arrays; d = b200bo_gp_dim(gp), n = b200bo_gp_n(gp).
 * A path owns copies of everything it evaluates: a later fit / append / lml on `gp` does not change it.  It lives
 * on gp's device and evaluates in fp64 whatever gp's precision. */
#define B200BO_MAX_PATHS 16

typedef struct b200bo_paths b200bo_paths; /* opaque: q posterior sample paths of one fitted GP */

/* 1 <= q <= B200BO_MAX_PATHS, L >= 1.  One solve of K v = r per path, O(N^2 q). */
int b200bo_paths_create(b200bo_gp* gp, int q, int L, const double* omega, const double* b, const double* w,
                        const double* eps, b200bo_paths** out);
void b200bo_paths_destroy(b200bo_paths* paths);
/* out: (m,q) host, path values at the rows of Xc (m,d) host, in data units.  A row's value depends on its
 * coordinates only (not on m, its position or the launch geometry). */
int b200bo_paths_eval(b200bo_paths* paths, const double* Xc, int64_t m, double* out);
/* Row mode of the batched refinement (one L-BFGS-B run per path): out: (m,) host, out[i] = path path_idx[i] at row i,
 * bit-equal to column path_idx[i] of b200bo_paths_eval on that row.  path_idx: (m,) host, every entry in [0, q), else
 * B200BO_ERR_ARG.  Costs one path per row instead of q. */
int b200bo_paths_eval_rows(b200bo_paths* paths, const double* Xc, const int* path_idx, int64_t m, double* out);
/* Row mode with the analytic input gradient: val[i] = path path_idx[i] at row i (bit-equal to
 * b200bo_paths_eval_rows), grad[i*d + j] = d val[i] / d x_ij (0 for a B200BO_XFORM_ROUND dimension).  val: (m,),
 * grad: (m,d) host.  path_idx as above. */
int b200bo_paths_grad_rows(b200bo_paths* paths, const double* Xc, const int* path_idx, int64_t m, double* val,
                           double* grad);
/* Per path p, ranks -path_p on the rows of Xc with the semantics of b200bo_acq_argmin_topk: best_val[p], best_idx[p]
 * (np.argmin), topk_val[p*k + i], topk_idx[p*k + i] (np.argsort order).  Large batches are streamed in chunks. */
int b200bo_paths_argmin_topk(b200bo_paths* paths, const double* Xc, int64_t m, int k, double* best_val,
                             int64_t* best_idx, double* topk_val, int64_t* topk_idx);
/* Throughput mode as b200bo_acq_argmin_topk_philox: candidates generated in the kernel from (seed, global index);
 * best_x: (q,d), topk_x: (q,k,d) host - the winners' rows. */
int b200bo_paths_argmin_topk_philox(b200bo_paths* paths, uint64_t seed, const double* lo, const double* hi, int64_t m,
                                    int64_t index_base, int k, double* best_val, int64_t* best_idx, double* best_x,
                                    double* topk_val, int64_t* topk_idx, double* topk_x);
/* Trust-region source (TuRBO / SCBO, DESIGN.md 4.18): the centre with a random subset of coordinates redrawn in the box
 * [lo, hi].  Per (seed, global row r, column j):
 *   u_j  = the b200bo_paths_argmin_topk_philox coordinate over [lo_j, hi_j]   (counter (r_lo, r_hi, j/2, 0))
 *   v_j  = the same 53-bit uniform from counter (r_lo, r_hi, j/2, 1)
 *   f(r) = (o0 * d) >> 32, o0 the first word of counter (r_lo, r_hi, 0, 2)
 *   x_j  = (j == f(r) || v_j < p) ? u_j : center_j
 * p = 1 draws no mask: the candidates are bit-equal to b200bo_paths_argmin_topk_philox over [lo, hi].  lo, hi, center:
 * (d,) host, lo <= center <= hi and all finite; 0 <= p <= 1; else B200BO_ERR_ARG.  Outputs as the plain entry. */
int b200bo_paths_argmin_topk_philox_tr(b200bo_paths* paths, uint64_t seed, const double* lo, const double* hi,
                                       const double* center, double p, int64_t m, int64_t index_base, int k,
                                       double* best_val, int64_t* best_idx, double* best_x, double* topk_val,
                                       int64_t* topk_idx, double* topk_x);
/* Rows of the trust-region source for given global indices (idx < 0 -> NaN row).  out: (n_idx, d) host. */
int b200bo_philox_tr_rows(int device, uint64_t seed, const double* lo, const double* hi, const double* center,
                          double p, int d, const int64_t* idx, int64_t n_idx, double* out);
/* bound: (q,) host.  B_p = |y_mean| + y_std (sqrt(2 const_value / L) sum_l |w[l][p]| + const_value sum_i |v[i][p]|),
 * computed at creation: |path_p(x)| <= B_p for every x, since |cos| <= 1 and 0 <= const_value k <= const_value. */
int b200bo_paths_bound(const b200bo_paths* paths, double* bound);

/* ---- constrained Thompson sampling (SCBO rule: Eriksson & Poloczek, AISTATS 2021) ------------------------------
 * The reference raises NoValidPointRegisteredError in EI / PoI until a registered point is feasible
 * (R/bayes_opt/acquisition.py:888-896); this rule needs no feasible point.  sets[0] = paths of the target GP,
 * sets[j] (1 <= j < G) = paths of constraint GP j with bounds lb[j-1] <= ub[j-1] (+-inf allowed); path p of every set
 * is one joint draw.  Per candidate x and path p, with f = sets[0] path p at x and c_j = sets[j] path p at x:
 *   viol_p(x)  = sum_{j=1..G-1}, in j order, of (max(0, lb_j - c_j) + max(0, c_j - ub_j))   (0 iff lb_j <= c_j <= ub_j)
 *   merit_p(x) = f                              if viol_p(x) == 0
 *              = -T_p (1 + viol_p(x))           otherwise,  T_p = 2 B_p + 1 (B_p of sets[0], b200bo_paths_bound)
 * so every infeasible merit lies below every feasible one.  Adds, subtracts, max (NaN-propagating, as np.maximum)
 * and one multiply, in this order and without FMA contraction.  The selection entries rank -merit_p with the
 * semantics of b200bo_paths_argmin_topk.  G <= B200BO_MAX_GPS; every set on the same device with the same d and q,
 * else B200BO_ERR_ARG.  The scratch lives in sets[0]; the handles are not thread-safe. */
/* merit: (m,q) host; raw: (m,G,q) host or NULL - raw[i][g][p] = path p of sets[g] at row i. */
int b200bo_cpaths_eval(b200bo_paths* const* sets, int G, const double* lb, const double* ub, const double* Xc,
                       int64_t m, double* merit, double* raw);
/* merit: (m,) host, merit[i] = merit of path path_idx[i] at row i, bit-equal to column path_idx[i] of
 * b200bo_cpaths_eval.  path_idx: (m,) host, every entry in [0, q), else B200BO_ERR_ARG. */
int b200bo_cpaths_eval_rows(b200bo_paths* const* sets, int G, const double* lb, const double* ub, const double* Xc,
                            const int* path_idx, int64_t m, double* merit);
int b200bo_cpaths_argmin_topk(b200bo_paths* const* sets, int G, const double* lb, const double* ub, const double* Xc,
                              int64_t m, int k, double* best_val, int64_t* best_idx, double* topk_val,
                              int64_t* topk_idx);
int b200bo_cpaths_argmin_topk_philox(b200bo_paths* const* sets, int G, const double* lb, const double* ub,
                                     uint64_t seed, const double* lo, const double* hi, int64_t m, int64_t index_base,
                                     int k, double* best_val, int64_t* best_idx, double* best_x, double* topk_val,
                                     int64_t* topk_idx, double* topk_x);
/* The same over the trust-region source of b200bo_paths_argmin_topk_philox_tr (SCBO). */
int b200bo_cpaths_argmin_topk_philox_tr(b200bo_paths* const* sets, int G, const double* lb, const double* ub,
                                        uint64_t seed, const double* lo, const double* hi, const double* center,
                                        double p, int64_t m, int64_t index_base, int k, double* best_val,
                                        int64_t* best_idx, double* best_x, double* topk_val, int64_t* topk_idx,
                                        double* topk_x);

/* Duration (ms) of the most recent fused predict+acquisition kernel launched through a
 * device or host entry point on this thread, measured with CUDA events on its stream.  With selection-only pruning
 * (DESIGN.md 4.9) it includes the bound pass and the sort; the selection merge is outside it either way.
 * Synchronises on the stop event. */
int b200bo_last_kernel_ms(float* ms);

/* Candidates of the most recent fused predict+acquisition call on this thread (a streamed host batch: all its chunks)
 * and how many of them went through the N^2 term.  Fewer than all when selection-only pruning skipped candidates whose
 * acquisition bound cannot reach the top-k (DESIGN.md 4.9).  Synchronises on the stop event. */
int b200bo_last_prune_stats(int64_t* evaluated, int64_t* total);

/* Where the kernel time of the most recent pruned launch on this thread went (a streamed or split batch: its last
 * launch), from CUDA events recorded between the stages on the call's stream: ms[0] bound pass, ms[1] sort,
 * ms[2] lead (the first tiles in bound order, split across SMs), ms[3] refine (leading-row-block bound, and its
 * levels), ms[4] final (exact evaluation of the refine survivors, split across SMs), ms[5] the whole-tile kernel in
 * bound order.  ms[2..4]
 * are 0 when the refine stages did not run (B200BO_PRUNE_REFINE=0, DESIGN.md 4.9).  *refined = candidates that went
 * through the refine stage (all launches of the call).  B200BO_ERR_STATE when the launch was not pruned.  Synchronises
 * on the stop event; nothing is read back unless this is called. */
int b200bo_last_prune_stage_ms(float ms[6], int64_t* refined);

/* The refine levels of the most recent pruned launch on this thread (DESIGN.md 4.9): *ms = their time (part of
 * ms[3] of b200bo_last_prune_stage_ms), *levels = how many ran (1 whenever the refine stages ran, else 0),
 * passed[0] = candidates the refine stage let through (more than 16384: the tile kernel took over and the level
 * evaluated nothing), passed[1 + l] = those level l let through; passed has room for 5.  B200BO_ERR_STATE when the
 * launch was not pruned.  Synchronises on the stop event. */
int b200bo_last_prune_levels(float* ms, int64_t passed[5], int* levels);

/* The direct bound pass of selection-only pruning alone (the one the selection runs for Matern-0.5; EI, UCB, PoI,
 * LogEI or LogPoI on one GP; 1 <= m <= INT_MAX device rows d_Xc):
 * d_key[i] = the order key (key_nan_last of select.cuh) of a lower bound on candidate i's closure value -acq, 0 for a
 * candidate that is never pruned; d_kmax[i] (nullable) = max_j |k(x_i, X_j)| in normalised units.  Enqueued on
 * `stream`, not synchronised.  For checking the bound against exact values. */
int b200bo_acq_prune_bound_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key, double* d_kmax,
                               void* stream);
/* The Gram bound pass of pruning (distances on the fp64 tensor pipe, DESIGN.md 4.9), as the selection uses it for
 * every covariance but Matern-0.5: per candidate a key no larger than the key of its exact value, the interval
 * d_mu[2i], d_mu[2i+1] (nullable, normalised units) that holds its exact K* alpha_, and d_kmax_lb (nullable) <= its
 * max_i |K*_i|.  B200BO_ERR_UNSUPPORTED for Matern-0.5. */
int b200bo_acq_prune_bound_gram_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key,
                                    double* d_mu, double* d_kmax_lb, void* stream);
/* The same with the covariance in fp32 (DESIGN.md 4.9): the same outputs and guarantees, with a wider mu interval.
 * The selection runs it when A1 constv 2^-24 <= 1e-3 (A1 = sum |alpha_|), see b200bo_acq_prune_bound_pass. */
int b200bo_acq_prune_bound_gram32_dev(const b200bo_acq* spec, const double* d_Xc, int64_t m, uint64_t* d_key,
                                      double* d_mu, double* d_kmax_lb, void* stream);
/* *pass = the bound pass a pruned selection of this spec's GP runs: 0 direct (Matern-0.5), 1 fp64 Gram, 2 fp32 Gram
 * (B200BO_PRUNE_BOUND=auto|f64|f32, read per call).  Builds the Gram operand if needed and synchronises `stream`. */
int b200bo_acq_prune_bound_pass(const b200bo_acq* spec, int* pass, void* stream);
/* The fp32 covariance of the fp32 Gram pass on n fp32 arguments r^2 (device): d_k[i], and d_z[i] (nullable) the
 * magnitude of its exp argument.  For tests of the margin. */
int b200bo_cov_f32_dev(int family, int nu, const float* d_r2, int64_t n, float* d_k, float* d_z, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200BO_H */

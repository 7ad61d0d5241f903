/*
 * bkm_b200.h — C ABI of the GPU-native KMeans hot path (libbkm_b200.so; built for H100, sm_90a).
 *
 * This is the drop-in boundary for the per-chunk operators that the reference
 * (mrocklin/dask-ml) invokes from its task graph.  dask-ml has no FFI layer of its
 * own; the callables replaced here are the ones its graph calls per row-chunk:
 *
 *   reference per-chunk callable                                  replaced by
 *   ------------------------------------------------------------  -------------------------
 *   sklearn.metrics.pairwise_distances_argmin_min(x, Y, ...)      bkm_lloyd_chunk (E-step half)
 *     dask_ml/metrics/pairwise.py:35-38                           bkm_assign_chunk
 *   _centers_dense(X, labels, n_clusters, distances)              bkm_lloyd_chunk (M-step half)
 *     dask_ml/cluster/k_means.py:572-582 (via da.atop :531-544)
 *   da.bincount(labels, minlength=k)  k_means.py:548              bkm_lloyd_chunk (counts)
 *   sum(r.to_delayed()) / counts, squared_norm(C - C')            bkm_finalize
 *     k_means.py:545-555
 *   metrics.pairwise_distances(x, Y).min(1)**2, p > U, where      bkm_assign_chunk + bkm_sample_chunk
 *     k_means.py:466-491, pairwise.py:55-66
 *   metrics.euclidean_distances(X, Y)  pairwise.py:69-97          bkm_transform_chunk
 *   da.isnull(X).any(), da.isinf(X).any()  k_means.py:179-180     bkm_check_finite
 *   pairwise_kernels(X_keep, X_rest) and the products with B of   bkm_kernel_colsum_chunk
 *     SpectralClustering.fit, cluster/spectral.py:237-270          bkm_nystrom_embed_chunk
 *   da.linalg.svd(X) + svd_flip of PCA / TruncatedSVD             bkm_gram_chunk + bkm_project_chunk
 *     decomposition/pca.py, truncated_svd.py
 *   X[y == c].mean(0) / .var(0) and _joint_log_likelihood of      bkm_class_moments_chunk + bkm_nb_jll_chunk
 *     GaussianNB, naive_bayes.py:32-122
 *   dask_glm's per-iteration X.dot(beta), family loglike /        bkm_glm_pass_chunk + bkm_gram_weighted_chunk
 *     gradient / hessian of LogisticRegression, LinearRegression,
 *     PoissonRegression, linear_model/glm.py:169-362
 *   the same per-iteration terms on sparse CSR blocks, which the      bkm_glm_csr_pass_chunk, bkm_csr_transpose_chunk,
 *     reference cannot take (linear_model/utils.py:34-53 appends a    bkm_csc_matvec_chunk,
 *     dense ones column to every block)                               bkm_gram_weighted_csr_chunk
 *   the Lloyd iterations, predict and transform of KMeans on sparse   bkm_csr_assign_chunk,
 *     CSR blocks, which the reference rejects (k_means.py:168)          bkm_csc_label_sums_chunk,
 *                                                                       bkm_sparse_pack_centers,
 *                                                                       bkm_sparse_finalize_step
 *   the mini-batch steps of PartialMiniBatchKMeans and the Nystrom      bkm_sparse_minibatch_step,
 *     passes of SpectralClustering on sparse CSR blocks, which the      bkm_csr_kernel_colsum_chunk,
 *     reference hands to scikit-learn / rejects                         bkm_csr_nystrom_embed_chunk
 *   da.linalg.svd_compressed's X.dot(omega), X.T.dot(q) and the        bkm_csr_panel_chunk, bkm_csc_panel_chunk
 *     projection of TruncatedSVD on sparse CSR blocks, which the
 *     reference densifies (decomposition/truncated_svd.py)
 *   X.mean(0) / .var(0) / .min(0) / .max(0), da.percentile and       bkm_colstats_chunk, bkm_radix_hist_chunk +
 *     the elementwise transforms of StandardScaler, MinMaxScaler,    bkm_radix_select_step, bkm_affine_chunk
 *     RobustScaler, preprocessing/data.py:24-221
 *   da.percentile at every reference and the per-column np.interp,   bkm_quantile_hist_chunk +
 *     ppf and cdf of QuantileTransformer, preprocessing/data.py:       bkm_quantile_select_step,
 *     224-312                                                          bkm_quantile_transform_chunk
 *   rng.normal X, X[:, idx].dot(beta[idx]) or da.dot(X, coef), then    bkm_make_glm_chunk
 *     rng.random < sigmoid(z), + noise, rng.poisson(exp(z)) of
 *     make_classification / make_regression / make_counts,
 *     datasets.py:24-73, 205-378
 *   check_random_state(seed).permutation(n) and x[idx] per block of    bkm_split_indices_chunk +
 *     ShuffleSplit / train_test_split, model_selection/_split.py:        bkm_gather_rows_chunk
 *     68-89, 321-360
 *   the elementwise graphs and reductions of accuracy_score,           bkm_metric_chunk
 *     log_loss, mean_squared_error, mean_absolute_error, r2_score,
 *     metrics/classification.py:11-150, metrics/regression.py:8-92
 *   scikit-learn's SimpleImputer._dense_fit / transform /             bkm_impute_stats_chunk,
 *     inverse_transform behind dask_ml/impute.py (np.ma.mean,            bkm_quantile_hist_masked_chunk,
 *     np.ma.median, the per-column mode, the masked fill and the          bkm_mode_*, bkm_impute_chunk
 *     indicator columns)
 *   da.unique / np.searchsorted / the sparse one-hot blocks of         bkm_distinct_chunk (+ bkm_mode_compact /
 *     LabelEncoder and OneHotEncoder, preprocessing/label.py:14-302,     bkm_mode_merge / bkm_mode_best),
 *     preprocessing/_encoders.py:18-244                                 bkm_encode_chunk, bkm_decode_chunk
 *   sklearn HashingVectorizer.transform per block of a 1-D dask array  bkm_text_tokens_chunk +
 *     of documents, feature_extraction/text.py:9-80 (tokenise, hash,     bkm_text_hash_chunk +
 *     sum duplicates, binary, normalize)                                 bkm_text_write_chunk
 *   the SGDClassifier / SGDRegressor / Perceptron / PassiveAggressive  bkm_sgd_order (host) +
 *     partial_fit of every block (_plain_sgd, one epoch), behind          bkm_sgd_block,
 *     linear_model/{stochastic_gradient,perceptron,passive_aggressive}    bkm_sgd_csr_block
 *     .py and _partial.py:39-100
 *   the MultinomialNB / BernoulliNB partial_fit counts (Y^T X) and       bkm_class_counts_chunk,
 *     the safe_sparse_dot(X, W^T) + b of their predict methods, behind    bkm_csc_class_counts_chunk,
 *     PartialMultinomialNB / PartialBernoulliNB (naive_bayes.py:125-134   bkm_nb_linear_jll_chunk,
 *     and _partial.py)                                                    bkm_nb_csr_jll_chunk
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only; no torch / C++ types.
 *   - every pointer is a DEVICE pointer unless its name ends in _host.
 *   - return 0 on success, negative BKM_E* for argument errors, positive values are
 *     forwarded cudaError_t codes.  Nothing throws across the ABI.
 *   - nothing allocates: the caller owns every buffer (sizes from the *_bytes helpers).
 *   - all work is enqueued asynchronously on `stream` (a cudaStream_t passed as void*).
 *   - X chunks are row-major (C order), `ldx` = row pitch in ELEMENTS (>= d).
 *   - There is NO CPU fallback: on a box without a GPU the compute entry points return
 *     a CUDA error (the library still loads, so symbol checks work without a driver).
 */
#ifndef BKM_B200_H
#define BKM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BKM_VERSION 200
/* Entry points added since BKM_VERSION 200 without changing an existing one raise the minor number:
 * 1 = bkm_split_indices_chunk, bkm_gather_rows_chunk, bkm_metric_workspace_bytes, bkm_metric_chunk
 * 2 = bkm_impute_stats_workspace_bytes, bkm_impute_stats_chunk, bkm_quantile_hist_masked_chunk, bkm_mode_count_chunk,
 *     bkm_mode_best_workspace_bytes, bkm_mode_best, bkm_mode_compact, bkm_mode_merge, bkm_impute_chunk
 * 3 = bkm_distinct_chunk, bkm_encode_chunk, bkm_decode_chunk
 * 4 = bkm_text_workspace_bytes, bkm_text_tokens_chunk, bkm_text_hash_chunk, bkm_text_write_chunk
 * 5 = bkm_glm_csr_workspace_bytes, bkm_glm_csr_pass_chunk, bkm_csr_transpose_workspace_bytes, bkm_csr_transpose_chunk,
 *     bkm_csc_matvec_workspace_bytes, bkm_csc_matvec_chunk, bkm_gram_weighted_csr_workspace_bytes,
 *     bkm_gram_weighted_csr_chunk
 * 6 = bkm_csr_panel_chunk, bkm_csc_panel_workspace_bytes, bkm_csc_panel_chunk
 * 7 = bkm_csr_assign_workspace_bytes, bkm_csr_assign_chunk, bkm_csc_label_sums_workspace_bytes,
 *     bkm_csc_label_sums_chunk, bkm_sparse_pack_workspace_bytes, bkm_sparse_pack_centers, bkm_sparse_finalize_step
 * 8 = bkm_csr_kernel_colsum_workspace_bytes, bkm_csr_kernel_colsum_chunk, bkm_csr_nystrom_embed_chunk,
 *     bkm_sparse_minibatch_step
 * 9 = bkm_sgd_order, bkm_sgd_block, bkm_sgd_csr_block
 * 10 = bkm_class_counts_chunk, bkm_csc_class_counts_chunk, bkm_nb_linear_jll_chunk, bkm_nb_csr_jll_chunk */
#define BKM_VERSION_MINOR 10

/* element types of X */
#define BKM_F32 0
#define BKM_F64 1
#define BKM_BF16 2   /* bfloat16 rows (16-byte row pitch); distances / min_d2 outputs are float32 */

/* error codes (negative) */
#define BKM_OK            0
#define BKM_EINVAL       -1   /* bad argument (null pointer, n<0, d<=0, k<=0, ldx<d ...) */
#define BKM_EDTYPE       -2   /* unsupported x_dtype */
#define BKM_EUNSUPPORTED -3   /* shape not supported by any kernel on this device */
#define BKM_EWORKSPACE   -4   /* workspace too small */
#define BKM_EALIGN       -5   /* pointer alignment requirement violated */

/* flags */
#define BKM_FLAG_FORCE_SIMT   1   /* never use the tensor-core path (exact-fp32 CUDA-core kernel) */
#define BKM_FLAG_FORCE_TC     2   /* fail with BKM_EUNSUPPORTED instead of falling back to SIMT */
#define BKM_FLAG_NO_RECHECK   4   /* skip the float64 re-check of near-tie rows */
#define BKM_FLAG_FIRST_CHUNK  8   /* bkm_lloyd_chunk: OVERWRITE sums / counts / inertia (first chunk of an iteration)
                                     instead of accumulating: saves the memsets of the step */
#define BKM_FLAG_COUNTS_F64  16   /* bkm_lloyd_chunk: `counts` points to float64 (so that sums | counts | inertia are ONE
                                     float64 buffer for the per-iteration all-reduce) */

int bkm_version(void);
const char* bkm_error_string(int code);

/* Device facts needed by the host: SM count and compute capability. */
int bkm_device_info(int device, int* sm_count, int* cc_major, int* cc_minor);

/* Which kernel family a (d, k, dtype, flags) problem dispatches to:
 * 0 = generic CUDA-core kernel (any d/k, fp32/fp64), 1 = wgmma tensor-core path (split-fp16 x3 product, fp32
 * accumulate; d <= 64, k <= 256), 2 = streaming CUDA-core kernel for tiny k*d (HBM-bound shapes: d <= 16, k <= 32).
 * <0 = error. */
int bkm_kernel_family(int d, int k, int x_dtype, int flags);

/* ---- centre pack -------------------------------------------------------------------
 * Kernels read the centres from an opaque "pack" built on the device from the float64
 * centres (the reference keeps centres in float64 from iteration 2 on: k_means.py:551-552).
 * The pack holds the layouts each kernel family wants (padded fp32/fp64 rows and ||c||^2 for
 * the CUDA-core kernels; -2sc split into fp16 hi/lo operand tiles for the tensor cores) plus the
 * float64 originals used by the near-tie re-check. */
int bkm_centers_pack_bytes(int k, int d, int x_dtype, size_t* out);
int bkm_pack_centers(const double* centers64, int k, int d, int x_dtype,
                     void* pack, size_t pack_bytes, void* stream);

/* Scratch for per-CTA partial sums / counts / inertia of one chunk call.  The first 8 KB are a PERSISTENT header (the
 * cluster -> warp balance table the label-indexed M-step pass leaves for the next call): zero them once when the buffer
 * is allocated and otherwise leave them alone; everything behind is overwritten by every call. */
int bkm_workspace_bytes(int64_t n, int d, int k, int x_dtype, size_t* out);

/* ---- fused E+M step for one row chunk ----------------------------------------------
 * replaces: pairwise_distances_argmin_min (pairwise.py:35-38) + _centers_dense
 * (k_means.py:572-582) + da.bincount (k_means.py:548) for ONE chunk.
 *   labels   [n]    int32  out : argmin_j ||x_i - c_j||^2, ties -> lowest j
 *   min_d2   [n]    x-dtype out, nullable : min_j ||x_i - c_j||^2 (clamped >= 0)
 *   sums     [k*d]  float64 ACCUMULATED (+=)  : sum of rows per label
 *   counts   [k]    int64   ACCUMULATED (+=)  : rows per label
 *   inertia  [1]    float64 ACCUMULATED (+=)  : sum_i min_d2_i
 * Accumulation across chunk calls on the same stream is in call order (the reference
 * folds chunk partials sequentially in chunk order, k_means.py:545-547). */
int bkm_lloyd_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                    const void* pack, int k,
                    int32_t* labels, void* min_d2,
                    double* sums, int64_t* counts, double* inertia,
                    void* workspace, size_t workspace_bytes, int flags,
                    const void* loop_state /* nullable, see bkm_loop_reset */, void* stream);

/* ---- E-step only (predict, final re-label, k-means|| cost) ---------------------------
 * replaces: pairwise_distances_argmin_min(X, centers[, squared]) per chunk.
 *   min_dist [n] x-dtype out, nullable: squared ? d^2 : sqrt(d^2)
 *   dist_sum [1] float64 ACCUMULATED: sum_i min_dist_i  (inertia, k_means.py:566; or
 *                 the k-means|| cost phi, k_means.py:466-469, with squared=1)
 *   labels nullable. */
int bkm_assign_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                     const void* pack, int k,
                     int32_t* labels, void* min_dist, int squared, double* dist_sum,
                     void* workspace, size_t workspace_bytes, int flags, void* stream);

/* ---- k-means|| Bernoulli sampling (k_means.py:472-491) -------------------------------
 * picked_i = (ell_over_phi * min_d2_i) > U_i with U_i = Philox4x32-10(seed, row_offset+i).
 * Appends the GLOBAL row index (row_offset+i) of every picked row to picked[] (unordered,
 * capacity `cap`), and adds the number of picked rows to *n_picked (may exceed cap: the
 * caller then retries with a bigger buffer). */
int bkm_sample_chunk(const void* min_d2, int64_t n, int x_dtype,
                     double ell_over_phi, uint64_t seed, uint64_t row_offset,
                     int64_t* picked, int64_t cap, int* n_picked, void* stream);

/* ---- k-means|| running minimum + cost (k_means.py:423-431, 466-469) ---------------------------------------------
 * run_min[i] = min(run_min[i], new_min[i]) (new_min nullable: cost only) and *phi_acc += sum_i run_min[i], in one
 * pass with a fixed reduction order.  min_d2 vectors have the dtype bkm_assign_chunk wrote them in (float32 for
 * float32 / bfloat16 rows, float64 for float64 rows): pass that as x_dtype. */
int bkm_min_fold_chunk(void* run_min, const void* new_min, int64_t n, int x_dtype, double* phi_acc, void* stream);

/* ---- transform: full (n,k) block of distances / kernel values -------------------------------------------------
 * replaces per chunk: metrics.euclidean_distances(X, Y[, squared])  pairwise.py:69-97  (KMeans.transform k_means.py:207-210)
 *                     metrics.rbf_kernel(X, Y, gamma) = exp(-gamma * d^2)  pairwise.py:131-139
 *   out [n][ld_out] x-dtype, row-major, ld_out >= k (so that callers can fill column blocks of a wider matrix):
 *   mode 0: sqrt(max(||x||^2 - 2 x.c + ||c||^2, 0))   mode 1: the squared distance   mode 2: exp(-gamma * d^2)
 * fp32 with d <= 64, k <= 256 runs on the tensor-core kernel (transform epilogue); other shapes on the CUDA cores. */
int bkm_transform_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                        const void* pack, int k, void* out, int64_t ld_out, int mode, double gamma, int flags,
                        void* stream);

/* ---- SpectralClustering: the two passes of the Nystrom embedding -------------------------------------------------
 * replace per chunk: pairwise_kernels(X_keep, X_rest, 'rbf') and every product with B in spectral.py:237-270
 * (A.sum(0) + B.sum(1), [A2; B2^T] . U . diag(S^-1/2) and the row normalisation of spectral.py:282).  The keep rows are
 * an ordinary centre pack (bkm_pack_centers with k = l).  With y_ij = max(||x_i - c_j||^2, 0) computed as in
 * bkm_transform_chunk:
 *   bkm_kernel_colsum_chunk  colsum[j] (l, float64) = sum_i exp(-gamma y_ij); OVERWRITTEN with BKM_FLAG_FIRST_CHUNK,
 *                            else ACCUMULATED (+=).  Rows, then per-CTA partials, are added in a fixed order:
 *                            bit-reproducible on one device.  workspace: bkm_workspace_bytes(n, d, l, x_dtype) bytes
 *                            (the same buffer as the chunk calls: its persistent header is left alone).
 *   bkm_nystrom_embed_chunk  out[i][0..k) = e_i / ||e_i||, e_i = sum_j exp(-gamma (y_ij - min_j y_ij)) W[j][0..k)
 *                            (W [l][k] row-major, x-dtype; out x-dtype with row pitch ld_out >= k).  The row shift
 *                            cancels in the normalisation and keeps fp32 from underflowing; a row with
 *                            gamma * min_j y_ij > 745.13 is written as NaN (the float64 reference gives 0 / 0 there).
 * fp32 rows with d <= 64, l <= 256 (embed: k <= 64) and 16-byte rows run on the tensor-core kernel; other shapes and
 * float64 rows on the CUDA cores (float64 throughout).  Honours BKM_FLAG_FORCE_SIMT / BKM_FLAG_FORCE_TC. */
int bkm_kernel_colsum_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack, int l,
                            double gamma, double* colsum, void* workspace, size_t workspace_bytes, int flags,
                            void* stream);
int bkm_nystrom_embed_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack, int l,
                            double gamma, const void* W, int k, void* out, int64_t ld_out, int flags, void* stream);

/* ---- PCA / TruncatedSVD: the two passes over row chunks (replace da.linalg.svd / svd_flip of
 * dask_ml/decomposition/pca.py and truncated_svd.py by a float64 Gram matrix and its eigendecomposition) -------------
 * Both widen the rows to float64, subtract the shift and multiply on the fp64 tensor cores (DMMA), so for every input
 * dtype the results are float64 sums of exact float64 products.  Any d, any row pitch ldx >= d.
 *   bkm_gram_chunk     colsum [d]    (+)= sum_i (x_i - shift)
 *                      gram   [d][d] (+)= sum_i (x_i - shift)(x_i - shift)^T   (full symmetric matrix, row-major)
 *                      OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  shift [d] float64 (device).  Per-CTA
 *                      partials are added in a fixed order: two calls with the same inputs give the same bits.
 *                      workspace: bkm_gram_workspace_bytes(n, d) bytes, any content.
 *   bkm_project_chunk  out [n][ldo] = (x - shift) W^T, out_dtype BKM_F32 or BKM_F64 (out nullable; shift nullable:
 *                      no shift), W [k][d] float64 row-major.  colmax (nullable) [k] records of 32 bytes
 *                      {double absmax, int64 row, double value, uint64 lock}: per column j the largest |out_ij| over
 *                      the chunk, its lowest GLOBAL row (row_offset + i) and the signed value, folded into the record
 *                      (larger |value| wins, equal |value| -> lower row).  Initialise records to {-1, -1, 0, 0}. */
int bkm_gram_workspace_bytes(int64_t n, int d, size_t* out);
int bkm_gram_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift, double* colsum,
                   double* gram, void* workspace, size_t ws_bytes, int flags, void* stream);
int bkm_project_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift,
                      const double* W, int k, void* out, int64_t ldo, int out_dtype, void* colmax, int64_t row_offset,
                      int flags, void* stream);

/* ---- GaussianNB: the fit passes and the predict pass over row chunks (replace the per-class X[y == c].mean / .var
 * and the K stacked elementwise passes of _joint_log_likelihood in dask_ml/naive_bayes.py) ---------------------------
 *   bkm_class_moments_chunk  cls [n] int32 class indices; rows with cls outside [0, K) are left out of every sum.
 *                      mode 0: sums [K][d] (+)= sum of the rows of class c, counts [K] float64 (+)= their number
 *                      mode 1: sums [K][d] (+)= sum of (x - theta_c)^2 over the rows of class c (theta [K][d] float64;
 *                              counts unused)
 *                      OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  float64 accumulators in a fixed order
 *                      (per-CTA row groups, then groups, then row splits): two calls with the same inputs give the
 *                      same bits.  workspace: bkm_nb_workspace_bytes(n, d, K) bytes, any content.
 *   bkm_nb_jll_chunk   jll_ic = logc_c - 1/2 sum_j (x_ij - theta_cj)^2 inv_sigma_cj (theta, inv_sigma [K][d], logc [K]
 *                      float64; all finite except logc, where NaN marks a class whose log-likelihood is NaN).
 *                      labels [n] (nullable): arg-max over c, lowest c on exact ties, the first NaN class if any.
 *                      out [n][ldo] float64 (nullable): jll - (log sum_c exp(jll - max) + max), exponentiated when
 *                      exp_out; a row with any NaN jll is NaN throughout.  fp32 / bf16 rows are computed in fp32; a row
 *                      whose best class is not ahead of every other class by the fp32 error bound is re-decided in
 *                      float64 (skipped with BKM_FLAG_NO_RECHECK) and counted into n_deferred (int32, nullable,
 *                      ACCUMULATED).  float64 rows are computed in float64.  Any d, any row pitch ldx >= d. */
int bkm_nb_workspace_bytes(int64_t n, int d, int K, size_t* out);
int bkm_class_moments_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* cls, int K,
                            int mode, const double* theta, double* sums, double* counts, void* workspace,
                            size_t ws_bytes, int flags, void* stream);
int bkm_nb_jll_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* theta,
                     const double* inv_sigma, const double* logc, int K, int32_t* labels, double* out, int64_t ldo,
                     int exp_out, int* n_deferred, int flags, void* stream);

/* ---- PartialMultinomialNB / PartialBernoulliNB: the count pass of partial_fit and the predict pass, on dense row
 * chunks and on CSR blocks (replace scikit-learn's safe_sparse_dot(Y^T, X) in _count and safe_sparse_dot(X, W^T) + b in
 * _joint_log_likelihood) -------------------------------------------------------------------------------------------
 * f(x) is x, or 1.0 where x > threshold and 0.0 elsewhere when `binarize` is nonzero (scikit-learn's binarize; for CSR
 * blocks an entry that is not above the threshold is dropped, as scipy drops the zeros binarize makes).
 *   bkm_class_counts_chunk      fc [K][d] (+)= sum_{i: cls_i = c} w_i f(x_ij),  cc [K] (+)= sum_{i: cls_i = c} w_i, w [n]
 *                               float64 (nullable: w_i = 1).  cls, the order of the sums, OVERWRITE / ACCUMULATE and the
 *                               workspace (bkm_nb_workspace_bytes) are those of bkm_class_moments_chunk mode 0.
 *   bkm_csc_class_counts_chunk  fcT [p][K] (+)= the same sums over the transpose of one CSR block (bkm_csr_transpose_chunk),
 *                               each (feature, class) sum in ascending row order; labels [n] int32 class indices (outside
 *                               [0, K) skipped).  Workspace: bkm_csc_label_sums_workspace_bytes(p, nnz, K) bytes.
 *   bkm_nb_linear_jll_chunk     jll_ic = b_c + sum_j f(x_ij) W_cj  (W [K][d], b [K] float64), float64 products on the fp64
 *                               tensor cores (0 * -inf = NaN, as BLAS).  Any d, any row pitch ldx >= d.
 *   bkm_nb_csr_jll_chunk        the same for one CSR block over the stored entries only, WT [p][K] float64 row-major.
 *   Both: labels [n] int32 (nullable) = the arg-max over c (the first maximum; the first NaN class if any, as np.argmax);
 *   out [n][ldo] float64 (nullable) = jll (BKM_NB_JLL), jll - (log sum_c exp(jll - max) + max) (BKM_NB_LOG_PROBA) or its
 *   exp (BKM_NB_PROBA); a normalised row with a NaN jll or no finite maximum is NaN throughout.  The sums run in a fixed
 *   order: two calls with the same inputs give the same bits. */
#define BKM_NB_JLL        0
#define BKM_NB_LOG_PROBA  1
#define BKM_NB_PROBA      2
int bkm_class_counts_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* cls, int K,
                           const double* w, int binarize, double threshold, double* fc, double* cc, void* workspace,
                           size_t ws_bytes, int flags, void* stream);
int bkm_csc_class_counts_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int p,
                               int64_t nnz, const int64_t* plan, const int32_t* labels, int K, const double* w,
                               int binarize, double threshold, double* fcT, void* workspace, size_t ws_bytes, int flags,
                               void* stream);
int bkm_nb_linear_jll_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int binarize, double threshold,
                            const double* W, const double* b, int K, int32_t* labels, double* out, int64_t ldo,
                            int out_mode, int flags, void* stream);
int bkm_nb_csr_jll_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int p,
                         int64_t nnz, int binarize, double threshold, const double* WT, const double* b, int K,
                         int32_t* labels, double* out, int64_t ldo, int out_mode, int flags, void* stream);

/* ---- LogisticRegression / LinearRegression / PoissonRegression: the per-iteration passes of the solvers (replace
 * dask_glm's X.dot(beta) and the family's loglike / gradient / hessian, linear_model/glm.py) ------------------------
 *   bkm_glm_pass_chunk  eta_i = x_i . beta[0:d] + beta[d]  (beta [d + 1] float64; rows widened to float64, float64
 *                      arithmetic).  family 0 logistic (mu = sigmoid(eta), loss = softplus(eta) - y eta, r = mu - y,
 *                      w = mu (1 - mu)), 1 normal (mu = eta, loss = (y - eta)^2, r = 2 (mu - y), w = 2), 2 poisson
 *                      (mu = exp(eta), loss = mu - y eta, r = mu - y, w = mu; exp overflows to +inf above 709.78).
 *                      mode 0 (gradient): grad [d + 2] (+)= [sum r_i x_i | sum r_i | sum loss_i]   (y [n] float64)
 *                      mode 1 (Newton):   the same, and w [n] = w_i, hrow [d + 1] (+)= [sum w_i x_i | sum w_i]
 *                      mode 2 (predict):  out [n] float64 = mu_i          mode 3 (labels): out [n] uint8 = mu_i > 0.5
 *                      (the predict modes take no y and accumulate nothing).  OVERWRITTEN with BKM_FLAG_FIRST_CHUNK,
 *                      else ACCUMULATED.  Per-CTA partials are added in a fixed order (no float atomics): two calls
 *                      with the same inputs give the same bits.  Any d, any row pitch ldx >= d.  One launch.
 *                      workspace: bkm_glm_workspace_bytes(n, d) bytes, any content (unused by the predict modes).
 *   bkm_gram_weighted_chunk  gram [d][d] (+)= sum_i w_i x_i x_i^T (w [n] float64; full symmetric matrix), the
 *                      Hessian block of a Newton step.  The kernel of bkm_gram_chunk without shift and column sums,
 *                      the weight applied to one operand as the rows are widened; same order guarantee.
 *                      workspace: bkm_gram_workspace_bytes(n, d) bytes. */
int bkm_glm_workspace_bytes(int64_t n, int d, size_t* out);
int bkm_glm_pass_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* y, const double* beta,
                       int family, int mode, double* grad, double* hrow, double* w, void* out, void* workspace,
                       size_t ws_bytes, int flags, void* stream);
int bkm_gram_weighted_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* w, double* gram,
                            void* workspace, size_t ws_bytes, int flags, void* stream);

/* ---- The same passes on one sparse CSR block: crow [n + 1] int64 row pointers, col [nnz] int64 column indices, val
 * [nnz] values of val_dtype BKM_F32 or BKM_F64, widened to float64.  Every sum runs in a fixed order (no float atomics):
 * two calls with the same inputs give the same bits.  ---------------------------------------------------------------
 *   bkm_glm_csr_pass_chunk  eta_i = sum_k val_k beta[col_k] + beta[d], the families and modes of bkm_glm_pass_chunk.
 *                      Modes 0 / 1 write r [n] = r_i (and w [n] = w_i) for the column pass and set grad[d] = sum r_i,
 *                      grad[d + 1] = sum loss_i (and hrow[d] = sum w_i); grad[0:d] and hrow[0:d] are the column pass's.
 *                      Modes 2 / 3 write out as bkm_glm_pass_chunk.  Rows without entries are legal.  Column indices
 *                      outside [0, d) are skipped.  OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  One launch.
 *                      workspace: bkm_glm_csr_workspace_bytes(n) bytes, any content.
 *   bkm_csr_transpose_chunk  the block's CSC: colptr [d + 1] int64, rows [nnz] int32 (strictly ascending within each
 *                      column), vals [nnz] in val_dtype; n, nnz < 2^31 (else BKM_EUNSUPPORTED).  plan: int64 [status (4) |
 *                      the column segments that the two calls below read], status = [nonzero when a column index is
 *                      outside [0, d), not strictly above its predecessor in the row, or crow is not a valid row pointer
 *                      array | segments | Gram slots (n_slots below) | longest column].  plan_bytes and the workspace
 *                      (any content) from bkm_csr_transpose_workspace_bytes.  A CUB radix sort and five small launches.
 *   bkm_csc_matvec_chunk  out1[j] (+)= sum over column j's entries, in ascending row order, of v1[row] val (and out2 from
 *                      v2 when v2 is not null): the first d entries of grad / hrow.  A column of more than 2048 entries
 *                      is summed in segments whose partials are added in segment order.  One launch.  workspace:
 *                      bkm_csc_matvec_workspace_bytes(d, nnz) bytes, any content.
 *   bkm_gram_weighted_csr_chunk  gram [d][d] (+)= sum_i w_i x_i x_i^T (w [n] float64; the full matrix), each term
 *                      (w_i x_ij) x_ik, for d <= 12288 (else BKM_EUNSUPPORTED).  Column j's entries are walked in row order
 *                      in runs of up to 64 Ki entries; the runs of a longer column are added in run order.  One launch.
 *                      The work is sum_i nnz_i^2.  workspace: bkm_gram_weighted_csr_workspace_bytes(d, n_slots) bytes,
 *                      any content, n_slots = status[2] of the block's plan. */
int bkm_glm_csr_workspace_bytes(int64_t n, size_t* out);
int bkm_glm_csr_pass_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int d,
                           int64_t nnz, const double* y, const double* beta, int family, int mode, double* r, double* w,
                           double* grad, double* hrow, void* out, void* workspace, size_t ws_bytes, int flags,
                           void* stream);
int bkm_csr_transpose_workspace_bytes(int64_t n, int d, int64_t nnz, size_t* ws_bytes, size_t* plan_bytes);
int bkm_csr_transpose_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int d,
                            int64_t nnz, int64_t* colptr, int32_t* rows, void* vals, int64_t* plan, size_t plan_bytes,
                            void* workspace, size_t ws_bytes, void* stream);
int bkm_csc_matvec_workspace_bytes(int d, int64_t nnz, size_t* out);
int bkm_csc_matvec_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int d,
                         int64_t nnz, const int64_t* plan, const double* v1, const double* v2, double* out1,
                         double* out2, void* workspace, size_t ws_bytes, int flags, void* stream);
int bkm_gram_weighted_csr_workspace_bytes(int d, int64_t n_slots, size_t* out);
int bkm_gram_weighted_csr_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                int d, int64_t nnz, const int64_t* colptr, const int32_t* rows, const void* vals,
                                const int64_t* plan, int64_t n_slots, const double* w, double* gram, void* workspace,
                                size_t ws_bytes, int flags, void* stream);

/* ---- TruncatedSVD on sparse CSR blocks: the products of a block with a dense float64 panel (replace da.linalg's
 * svd_compressed power iterations X (X^T Q) and the projection X V^T, which the reference runs on dense blocks) --------
 * The block is given as for the linear models above (crow / col / val, or its transpose from bkm_csr_transpose_chunk).
 * Values are widened to float64; every sum runs in a fixed order (no float atomics): two calls with the same inputs give
 * the same bits.
 *   bkm_csr_panel_chunk  out [n][ldo] = X W, W [p][l] float64 row-major, out_dtype BKM_F32 or BKM_F64, any l >= 1.
 *                      Each out_ic adds row i's entries in stored order (ascending column for a canonical block) by fma;
 *                      column indices outside [0, p) are skipped.  colmax (nullable) [l] records of bkm_project_chunk's
 *                      format: per column the largest |out_ic| with its lowest GLOBAL row (row_offset + i) and the signed
 *                      value, folded into the record.  out nullable (the epilogue only).  One launch, no workspace.
 *   bkm_csc_panel_chunk  out [p][l] (+)= X^T P, P [n][l] float64 row-major, over the block's transpose and its plan:
 *                      each out_jc adds column j's entries in ascending row order; a column of more than 2048 entries is
 *                      summed in segments whose partials are added in segment order by the last segment to finish.
 *                      OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  One launch.  workspace:
 *                      bkm_csc_panel_workspace_bytes(p, nnz, l) bytes, any content: 2 (nnz / 2048 + 1) l float64 segment
 *                      partials, then p uint32 tickets (cleared by the call). */
int bkm_csr_panel_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int p,
                        int64_t nnz, const double* W, int l, void* out, int64_t ldo, int out_dtype, void* colmax,
                        int64_t row_offset, void* stream);
int bkm_csc_panel_workspace_bytes(int p, int64_t nnz, int l, size_t* out);
int bkm_csc_panel_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int p,
                        int64_t nnz, const int64_t* plan, const double* P, int l, double* out, void* workspace,
                        size_t ws_bytes, int flags, void* stream);

/* ---- KMeans on sparse CSR blocks: the E-step, the M-step sums and the centre update on transposed centres -----------
 * The block is given as for the linear models above.  Values are widened to float64; every sum runs in a fixed order
 * (no float atomics): two calls with the same inputs give the same bits.  The centres live in a SPARSE PACK of
 * p k + k float64: CT [p][k] (the centres transposed, so that one entry of a row gathers k contiguous values), then
 * cn [k] = ||c_j||^2.  Only bkm_sparse_pack_centers and bkm_sparse_finalize_step write packs, with the same kernel.
 *   bkm_sparse_pack_centers   pack = the sparse pack of centres64 [k][p] float64.  cn_j sums c_jf^2 over f in a fixed
 *                      order.  workspace: bkm_sparse_pack_workspace_bytes(k, p) bytes, any content.
 *   bkm_csr_assign_chunk      d2_ij = max(||x_i||^2 - 2 x_i.c_j + cn_j, 0), ||x_i||^2 and x_i.c_j adding row i's
 *                      entries in stored order by fma (column indices outside [0, p) are skipped).  Any k >= 1, one
 *                      launch, no (n x k) intermediate.  mode:
 *                        BKM_SPARSE_ARGMIN  labels [n] int32 = arg-min_j (ties to the lowest j), min_out [n] float64 =
 *                          the minimum (d2, or its square root unless `squared`), dist_sum [1] float64 = the sum of
 *                          min_out, counts [k] float64 = the rows per cluster; all nullable.  dist_sum and counts are
 *                          OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED; they need the workspace
 *                          (bkm_csr_assign_workspace_bytes(n, k) bytes, any content).  n = 0 still writes them.
 *                        BKM_SPARSE_DIST / BKM_SPARSE_DIST2  out [n][ldo] (ldo >= k) = sqrt(d2) / d2 in out_dtype
 *                          (BKM_F32 or BKM_F64).
 *                      loop_state (nullable): a no-op once the loop of bkm_loop_reset is done.
 *   bkm_csc_label_sums_chunk  sumsT [p][k] (+)= X^T onehot(labels) over the block's transpose and plan: entry (row, v)
 *                      of column j adds v to sumsT[j][labels[row]] (labels outside [0, k) are skipped); each (j, c) sum
 *                      runs in ascending row order, a column of more than 2048 entries in segments added in segment
 *                      order.  OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  k <= 25600.  workspace:
 *                      bkm_csc_label_sums_workspace_bytes(p, nnz, k) bytes, any content.  loop_state as above.
 *   bkm_sparse_finalize_step  the contract of bkm_finalize_step on the transposed layout: reduced = [p k sumsT |
 *                      k counts as float64 | inertia] of the iteration, C' = sumsT / max(counts, 1) (an empty cluster
 *                      gets 0), shift = sum_j sum_f (CT_fj - C'_fj)^2 (f, then j, in a fixed order) -> the loop state
 *                      and its history; pack_out (!= pack_in) = the sparse pack of C', written whether or not the
 *                      iteration converged (the loop then keeps pack_in, Q3).  A no-op once the loop is done.
 *                      workspace: bkm_sparse_pack_workspace_bytes(k, p) bytes. */
#define BKM_SPARSE_ARGMIN 0
#define BKM_SPARSE_DIST   1
#define BKM_SPARSE_DIST2  2
int bkm_sparse_pack_workspace_bytes(int k, int p, size_t* out);
int bkm_sparse_pack_centers(const double* centers64, int k, int p, double* pack, void* workspace, size_t ws_bytes,
                            void* stream);
int bkm_csr_assign_workspace_bytes(int64_t n, int k, size_t* out);
int bkm_csr_assign_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int p,
                         int64_t nnz, const double* pack, int k, int mode, int32_t* labels, double* min_out,
                         int squared, double* dist_sum, double* counts, void* out, int64_t ldo, int out_dtype,
                         void* workspace, size_t ws_bytes, int flags, const void* loop_state, void* stream);
int bkm_csc_label_sums_workspace_bytes(int p, int64_t nnz, int k, size_t* out);
int bkm_csc_label_sums_chunk(const int64_t* colptr, const int32_t* rows, const void* vals, int val_dtype, int p,
                             int64_t nnz, const int64_t* plan, const int32_t* labels, int k, double* sumsT,
                             void* workspace, size_t ws_bytes, int flags, const void* loop_state, void* stream);
int bkm_sparse_finalize_step(const double* reduced, const double* pack_in, double* pack_out, void* loop_state, int k,
                             int p, void* workspace, size_t ws_bytes, void* stream);

/* ---- PartialMiniBatchKMeans and SpectralClustering on sparse CSR blocks: the same conventions (float64, fixed order, no
 * float atomics, the same bits from two calls), over a sparse pack.
 *   bkm_csr_kernel_colsum_chunk  the contract of bkm_kernel_colsum_chunk for one CSR block against the sparse pack of
 *                      the l keep rows (bkm_sparse_pack_centers with k = l): colsum[j] (l, float64) = sum_i
 *                      exp(-gamma y_ij), y_ij = max(||x_i||^2 - 2 x_i.c_j + ||c_j||^2, 0) as in bkm_csr_assign_chunk.
 *                      Rows add in warp order, warps in CTA order, CTAs in CTA order.  OVERWRITTEN with
 *                      BKM_FLAG_FIRST_CHUNK, else ACCUMULATED (n = 0 still overwrites).  workspace:
 *                      bkm_csr_kernel_colsum_workspace_bytes(n, l) bytes, any content.
 *   bkm_csr_nystrom_embed_chunk  the contract of bkm_nystrom_embed_chunk: out_i = e_i / ||e_i||, e_i = sum_j
 *                      exp(-gamma (y_ij - m_i)) W_j, m_i = min_j y_ij, W [l][k] float64, out [n][ldo] (ldo >= k) in
 *                      out_dtype (BKM_F32 or BKM_F64); NaN where gamma m_i > 745.13.  Any l; e_i adds j in ascending
 *                      order by fma.  k <= 3000.
 *   bkm_sparse_minibatch_step  scikit-learn's _minibatch_update_sparse on the transposed layout: reduced = [p k sumsT |
 *                      k counts as float64 | inertia] of the batch, C' = (C w + S) (1 / (w + n)) where n > 0, else C
 *                      (explicit round-to-nearest float64, as bkm_minibatch_step), w' = w + n; pack_out (!= pack_in)
 *                      = the sparse pack of C', weights_out (!= weights_in) = w'.  workspace:
 *                      bkm_sparse_pack_workspace_bytes(k, p) bytes. */
int bkm_csr_kernel_colsum_workspace_bytes(int64_t n, int l, size_t* out);
int bkm_csr_kernel_colsum_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                int p, int64_t nnz, const double* pack, int l, double gamma, double* colsum,
                                void* workspace, size_t ws_bytes, int flags, void* stream);
int bkm_csr_nystrom_embed_chunk(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                int p, int64_t nnz, const double* pack, int l, double gamma, const double* W, int k,
                                void* out, int64_t ldo, int out_dtype, int flags, void* stream);
int bkm_sparse_minibatch_step(const double* reduced, const double* pack_in, const double* weights_in, double* pack_out,
                              double* weights_out, int k, int p, void* workspace, size_t ws_bytes, void* stream);

/* ---- StandardScaler / MinMaxScaler / RobustScaler: the fit passes and the transform pass over row chunks (replace
 * X.mean(0), X.var(0), X.min(0), X.max(0), da.percentile per column and the elementwise (X - m) / s of
 * dask_ml/preprocessing/data.py) ---------------------------------------------------------------------------------------
 *   bkm_colstats_chunk   per column j, in float64: acc [5][d] (+)= [sum (x - shift_j) | sum (x - shift_j)^2 over the
 *                        finite x | number of NaN | of +inf | of -inf]; minmax [2][d] = [min | max] over the non-NaN x
 *                        (+inf / -inf when there is none), folded with min / max.  shift [d] float64, nullable.
 *                        OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  CTA partials are folded in a fixed
 *                        order: two calls with the same inputs give the same bits.  One launch.
 *                        workspace: bkm_colstats_workspace_bytes(n, d) bytes, any content.
 *   bkm_radix_hist_chunk + bkm_radix_select_step   exact order statistics per column, T (even, <= 6) target ranks per
 *                        column: for target t the ranks floor(v) + (t & 1) of numpy's 'linear' virtual index
 *                        v = (m - 1) q[t / 2] over the m non-NaN values (both the last value when v >= m - 1, both
 *                        the first when v < 0).  Values map to order-preserving unsigned keys of 16 (bf16), 32 (fp32)
 *                        or 64 (fp64) bits, selected 8 bits per round: 2, 4 or 8 rounds.  Round r:
 *                          every chunk: bkm_radix_hist_chunk(..., state, T, r, hist) histograms the next digit of the
 *                            keys that carry each target's prefix (NaN rows skipped); hist [d][T][256] float64 counts,
 *                            ZEROED with BKM_FLAG_FIRST_CHUNK (set it on the first chunk of every round), else
 *                            ACCUMULATED.  Counts are integers: the sums are exact whatever the order, and all-reduce.
 *                          then: bkm_radix_select_step(hist, state, d, T, r, x_dtype, q_host) extends each target's
 *                            prefix by one digit on the device (round 0 also derives the ranks and sets nvalid).
 *                        state: bkm_radix_state_bytes(d, T) bytes, any content before round 0; after the last round
 *                        state [d][T] holds records of 32 bytes {uint64 key, double rank, double nvalid, int32 slot,
 *                        int32 pad}: `key` is the key of the target's order statistic, `nvalid` the column's non-NaN
 *                        count.  q_host [T / 2] float64 quantiles in [0, 1] (host memory, read at the call).
 *   bkm_affine_chunk     out [n][ld_out] = op2(op1(x, a), b) per element, op1: 0 none, 1 x - a_j, 2 x * a_j;
 *                        op2: 0 none, 1 / b_j, 2 + b_j (a, b [d] float64, values of the output dtype).  out_dtype
 *                        BKM_F32 (x fp32 or bf16) or BKM_F64; every operation is rounded once in the output dtype
 *                        (no FMA contraction), which is numpy's two-step expression.  Any ldx >= d, ld_out >= d. */
int bkm_colstats_workspace_bytes(int64_t n, int d, size_t* out);
int bkm_colstats_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* shift, double* acc,
                       double* minmax, void* workspace, size_t ws_bytes, int flags, void* stream);
int bkm_radix_state_bytes(int d, int T, size_t* out);
int bkm_radix_hist_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* state, int T, int round,
                         double* hist, int flags, void* stream);
int bkm_radix_select_step(double* hist, void* state, int d, int T, int round, int x_dtype, const double* q_host,
                          void* stream);
int bkm_affine_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* a, const double* b,
                     int op1, int op2, void* out, int64_t ld_out, int out_dtype, void* stream);

/* ---- QuantileTransformer: the fit selection and the transform pass over row chunks (replace da.percentile per
 * column at every reference and the per-column np.interp / ppf / cdf of dask_ml/preprocessing/data.py:224-312) ------
 *   bkm_quantile_hist_chunk + bkm_quantile_select_step   exact order statistics per column at T = 2 n_q target ranks:
 *                        for quantile i the ranks floor(v) and floor(v) + 1 of numpy's 'linear' virtual index
 *                        v = (m - 1) qf[i] over the m non-NaN values (both m - 1 when v >= m - 1), with the keys and
 *                        rounds of bkm_radix_hist_chunk.  The selection works on the column's sorted distinct ranks;
 *                        their prefixes after round r form a sorted, duplicate-free live list of
 *                        L <= cap(r) = min(T, 256^r) entries.  Round r:
 *                          every chunk: bkm_quantile_hist_chunk(..., state, n_q, r, hist) counts the next digit of the
 *                            keys whose prefix is live (NaN rows skipped); hist [d][cap(r)][256] float64 counts,
 *                            ZEROED with BKM_FLAG_FIRST_CHUNK (set it on the first chunk of every round), else
 *                            ACCUMULATED.  Counts are integers: the sums are exact whatever the order, and all-reduce.
 *                          then: bkm_quantile_select_step(hist, state, d, n_q, r, x_dtype, qf) extends each distinct
 *                            rank's prefix by one digit and builds the next live list, one CTA per column; round 0
 *                            also derives the ranks.  It overwrites hist.
 *                        qf [n_q] float64 ascending quantiles in [0, 1] (device memory).
 *                        state: bkm_quantile_state_bytes(d, n_q) bytes, any content before round 0.  Column j's record
 *                        starts at byte j * (16 + 80 n_q): {double nvalid, int32 R, int32 L}, then T records of 32 bytes
 *                        {uint64 key, double rank, double nvalid, int32 slot, int32 pad} whose first R hold the distinct
 *                        ranks in ascending order (after the last round `key` is the key of that order statistic), then
 *                        T uint64 live prefixes.  The caller may run column groups as views: X + j0, state + j0 stride.
 *   bkm_quantile_transform_chunk   out [n][ld_out] float64 per element, with the quantiles q = quantiles[j][0, n_q)
 *                        (float64, ascending, one row per column) and the references r [n_q] of column j:
 *                          forward (inverse 0): y = 0.5 (interp(x, q, r) - interp(-x, -q[::-1], -r[::-1])); y = 1 where
 *                            x + 1e-7 > q[n_q - 1], then y = 0 where x - 1e-7 < q[0] (that test in X's dtype: float32 for
 *                            fp32 and bf16 rows); out = clip(ppf(y), clip_lo, clip_hi);
 *                          inverse (inverse 1): c = cdf(x); out = interp(c, r, q), then q[n_q - 1] where c + 1e-7 > 1,
 *                            then q[0] where c - 1e-7 < 0;
 *                        interp is numpy's, every operation rounded once in float64; distribution 0 uniform (ppf the
 *                        identity on [0, 1], cdf a clip to [0, 1]), 1 normal (normcdfinv / normcdf).  NaN x gives NaN
 *                        (n_q > 1).  Any ldx >= d, ld_out >= d; the input is only read. */
int bkm_quantile_state_bytes(int d, int n_q, size_t* out);
int bkm_quantile_hist_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* state, int n_q,
                            int round, double* hist, int flags, void* stream);
int bkm_quantile_select_step(double* hist, void* state, int d, int n_q, int round, int x_dtype, const double* qf,
                             void* stream);
int bkm_quantile_transform_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const double* quantiles,
                                 const double* references, int n_q, int inverse, int distribution, double clip_lo,
                                 double clip_hi, double* out, int64_t ld_out, void* stream);

/* ---- centre update + shift (k_means.py:548-555), run after the cross-GPU allreduce ----
 *   C_new = sums / max(counts,1)[:,None]   (empty cluster -> zero vector, Q1)
 *   *shift = sum((C_old - C_new)^2)        (float64)                                  */
int bkm_finalize(const double* sums, const int64_t* counts, const double* centers_old,
                 double* centers_new, double* shift, int k, int d, void* stream);

/* ---- device-resident Lloyd loop (k_means.py:522-560 without a host round trip per iteration) -----------------
 * The reference reads the shift back to the client every iteration (k_means.py:552-559).  Here the stop test runs on
 * the device: a small LoopState {done, n_iter, tol, shift, shift history} lives in device memory; bkm_finalize_step
 * updates it, and every kernel of a bkm_lloyd_chunk call that was given the state returns at once when `done` is set.
 * The host enqueues iterations back to back and looks at the state every few iterations; iterations enqueued after
 * convergence are no-ops, so n_iter, the centres and the labels are exactly those of the reference's loop.
 *   bkm_loop_reset     done = 0, n_iter = 0, tol; shift_hist (device, nullable): shift of iteration i at [i]
 *   bkm_finalize_step  replaces bkm_finalize (+ bkm_pack_centers for the next iteration):
 *       reduced = [k*d sums | k counts as float64 | inertia]  (BKM_FLAG_COUNTS_F64; after the all-reduce)
 *       C' = sums / max(counts, 1); shift = ||centers_in - C'||_F^2; n_iter += 1
 *       shift < tol : done = 1, centers_out is not meaningful (the reference breaks BEFORE taking C' over, Q3)
 *       else        : centers_out = C' and `pack` is rebuilt from C'  (centers_in != centers_out: ping-pong)
 * Read the state back with a plain device->host copy of bkm_loop_state_bytes() bytes: {int32 done, int32 n_iter,
 * int32 hist_cap, int32 pad, float64 tol, float64 shift, pointer}. */
int bkm_loop_state_bytes(size_t* out);
int bkm_loop_reset(void* loop_state, double tol, double* shift_hist, int hist_cap, void* stream);
int bkm_finalize_step(const double* reduced, const double* centers_in, double* centers_out, void* loop_state,
                      int k, int d, int x_dtype, void* pack, size_t pack_bytes, void* stream);

/* ---- one mini-batch k-means step: replaces scikit-learn's _minibatch_update_dense -------------------------------
 * (sklearn/cluster/_k_means_minibatch.pyx, called by MiniBatchKMeans.partial_fit through _mini_batch_step) on the
 * result of one bkm_lloyd_chunk pass over the batch with BKM_FLAG_FIRST_CHUNK | BKM_FLAG_COUNTS_F64:
 *   reduced = [k*d sums S | k counts n as float64 | inertia]
 *   centers_out[j] = (centers_in[j] * weights_in[j] + S[j]) * (1 / (weights_in[j] + n[j]))   if n[j] > 0
 *                  = centers_in[j]                                                          otherwise
 *   weights_out[j] = weights_in[j] + n[j]
 * evaluated in float64 without FMA contraction, and `pack` rebuilt from centers_out (the bytes bkm_pack_centers
 * writes for them).  centers_in != centers_out and weights_in != weights_out: ping-pong buffers. */
int bkm_minibatch_step(const double* reduced, const double* centers_in, const double* weights_in, double* centers_out,
                       double* weights_out, int k, int d, int x_dtype, void* pack, size_t pack_bytes, void* stream);

/* ---- datasets.make_blobs, one block on the device (dask_ml/datasets.py:178-189) ---------------------------------
 * The reference generates every block independently from (centres, cluster_std, seed = block index) with
 * sklearn.datasets.make_blobs; this is the device-side equivalent of ONE block: label_i ~ U{0..k-1}, row_i =
 * centres[label_i] + cluster_std[label_i] * N(0, I), Philox4x32-10 streams keyed by `seed` with (row, feature pair)
 * counters (reproducible per block whatever GPU generates it; numpy's Mersenne-Twister stream is not reproduced).
 * X [n][ldx] x-dtype out, y [n] int64 out (nullable); centers [k][d] and cluster_std [k] float64 on the device. */
int bkm_make_blobs_chunk(void* X, int64_t* y, int64_t n, int d, int64_t ldx, int x_dtype, const double* centers,
                         const double* cluster_std, int k, uint64_t seed, void* stream);

/* ---- datasets.make_classification / make_regression / make_counts, one block on the device ----------------------
 * (dask_ml/datasets.py:24-73, 205-378).  The reference's dask streams cannot be reproduced, so the package defines its
 * own, and dask_ml_b200.datasets restates it in numpy for device=None (the two give the same X to rounding of the
 * math library and the same y except where it sits within ~1e-12 of a decision):
 *   host parameter draws, numpy RandomState rng (sklearn.utils.check_random_state(random_state)), in this order:
 *     make_regression:              coef from sklearn.datasets.make_regression(n_samples=<first block>, ..., rng),
 *                                   then key;
 *     make_classification / counts: key, then idx = rng.choice(n_features, n_informative) (with replacement),
 *                                   then beta = (rng.random_sample(n_features) - 1) * scale;
 *     key = the first 8 bytes (little-endian uint64) of rng.bytes(624 * 4).
 *   per-element draws: w = Philox4x32-10(key, counter = (row lo, row hi, j, tag)), row = the GLOBAL row index:
 *     tag 0  X[row, 2p], X[row, 2p+1] (j = p): u1 = (w0 + 1) / 2^32, u2 = w1 / 2^32, r = sqrt(-2 log u1),
 *            r * cospi(2 u2), r * sinpi(2 u2)   (the Box-Muller of bkm_make_blobs_chunk)
 *     tag 1  response uniforms (j = attempt): U = ((w0 >> 5) 2^26 + (w1 >> 6)) / 2^53, V = the same of (w2, w3)
 *     tag 2  noise normal of target t (j = t): the cosine normal of (w0, w1)
 *   z[t] = sum over the list, in list order, of x_f * c[f, t], x_f the value AS STORED in X's dtype, in float64 with
 *          correctly rounded steps (no FMA), starting from 0.0
 *   family 0 logistic:  y = U < 1 / (1 + exp(-z))                                   int64 [n]
 *   family 1 normal:    y[t] = (z[t] + bias) (+ noise * N_t if noise > 0)             float64 [n][n_targets]
 *   family 2 poisson:   y ~ numpy's legacy Poisson of lam = exp(z) (multiplication method for lam < 10, PTRS with
 *                       numpy's loggam for lam >= 10), each loop turn / attempt taking counter j = 0, 1, ...; a rate
 *                       that numpy rejects (NaN or above its lam maximum 9.223372006484771e18) ORs 1 into *flag and
 *                       writes y = 0                                                    int64 [n]
 * X [n][ldx] x-dtype out (BKM_F32 / BKM_F64); y out as above; row0 = the global index of the block's first row;
 * info [m][1 + n_targets] float64: the feature index, then its coefficient for every target (n_targets = 1 for
 * families 0 and 2); flag int32 (needed for family 2).  One launch: every X element is written once, and the
 * informative normals of a row are recomputed from their counters for z, so X is never read back. */
int bkm_make_glm_chunk(void* X, void* y, int64_t n, int d, int64_t ldx, int x_dtype, int64_t row0, int family,
                       const double* info, int m, int n_targets, double bias, double noise, uint64_t key, int* flag,
                       void* stream);

/* ---- train_test_split / ShuffleSplit: the passes over one row block (replace, per block,
 * check_random_state(seed).permutation(n) and x[idx] of dask_ml/model_selection/_split.py:68-89, 321-360) -----------
 * The split permutation.  numpy's Mersenne-Twister Fisher-Yates is serial, so the package defines its own permutation
 * of a block of c rows (1 <= c <= 2^31), a keyed bijection pi_seed : [0, c) -> [0, c) that is evaluated per position;
 * dask_ml_b200.model_selection restates it in numpy (permutation_indices), bit for bit:
 *   domain    w = max(1, ceil(ceil(log2 c) / 2)); the network permutes the 2w-bit values [0, 4^w), 4^w < 4c
 *   keys      for round r = 0 .. BKM_SPLIT_ROUNDS - 1 (64-bit wrapping arithmetic, the splitmix64 finaliser):
 *               z = seed + (r + 1) * BKM_SPLIT_KEY_STEP;  z = (z ^ (z >> 30)) * BKM_SPLIT_KEY_MUL1;
 *               z = (z ^ (z >> 27)) * BKM_SPLIT_KEY_MUL2;  z = z ^ (z >> 31);  k0_r = low 32 bits, k1_r = high 32 bits
 *   network   v = (L << w) | R;  every round, in order:  x = R ^ k0_r (32 bits);  p = x * BKM_SPLIT_ROUND_MUL (64 bits);
 *               f = (p >> 32) ^ (low 32 bits of p) ^ k1_r;  f = (f ^ (f >> 16)) * BKM_SPLIT_ROUND_MIX (32 bits);
 *               f = f ^ (f >> 15);  (L, R) <- (R, L ^ (f >> (32 - w)))
 *             a balanced Feistel network with Philox's multiply-hi/lo round function and a multiply-xorshift
 *             finaliser (the top w bits of the product alone are close to affine in R): a bijection of [0, 4^w)
 *   walk      pi_seed(i): v = i; do v = network(v) while v >= c.  The cycle of the network through a value below c
 *             returns to a value below c, so the walk ends; fewer than 4 applications are expected.
 * BKM_SPLIT_ROUNDS: a network on 2 or 4 bits has few round functions to choose from and mixes slowly whatever the
 * hash; 12 is the count at which the position-uniformity and pair-independence tests of
 * tests/test_model_selection_host.py pass (6 rounds fail them), and at which 10^6 seeds show no bias above 1e-3
 * relative for c = 3, 5, 8.
 *   bkm_split_indices_chunk  idx_out[i] = offset + pi_seed(start + i) for i < count (start + count <= c).  One launch.
 *   bkm_gather_rows_chunk    out row i = src row (idx[i] - idx_offset) for i < count.  Typeless: a row is row_bytes
 *                            bytes, pitches are in bytes, so rows of any dtype and 1-D arrays (row_bytes = the element
 *                            size) go through it.  Copies in units of 16 bytes when both base addresses, both pitches
 *                            and row_bytes allow, else 8, 4, 2 or 1.  An index outside [0, n_src) is a caller error
 *                            that is NOT detected (a build with -DBKM_DEBUG asserts on it).  One launch. */
#define BKM_SPLIT_ROUNDS    12
#define BKM_SPLIT_KEY_STEP  0x9E3779B97F4A7C15ull
#define BKM_SPLIT_KEY_MUL1  0xBF58476D1CE4E5B9ull
#define BKM_SPLIT_KEY_MUL2  0x94D049BB133111EBull
#define BKM_SPLIT_ROUND_MUL 0xD2511F53u
#define BKM_SPLIT_ROUND_MIX 0x7FEB352Du
int bkm_split_indices_chunk(uint64_t seed, int64_t c, int64_t start, int64_t count, int64_t offset, int64_t* idx_out,
                            void* stream);
int bkm_gather_rows_chunk(const void* src, int64_t n_src, int64_t row_bytes, int64_t ld_src_bytes, const int64_t* idx,
                          int64_t idx_offset, int64_t count, void* out, int64_t ld_out_bytes, void* stream);

/* ---- accuracy_score / log_loss / mean_squared_error / mean_absolute_error / r2_score: one reduction pass over a
 * pair of row chunks (replace the elementwise graphs and reductions of dask_ml/metrics/classification.py:11-150 and
 * regression.py:8-92) ------------------------------------------------------------------------------------------------
 *   bkm_metric_chunk   a, b: (n, m) contiguous row-major operands (m = 1 for 1-D), each of its own element type
 *                      (BKM_F32, BKM_F64, BKM_BF16 or one of the BKM_M_* codes below); w [n] float64 row weights,
 *                      nullable (all 1).  One read of both, float64 arithmetic.
 *                      BKM_METRIC_EQ       acc [2] (+)= [sum_i w_i [a_ij == b_ij for all j] | sum_i w_i]; two integer
 *                                          operands are compared as int64, any other pair as float64
 *                      BKM_METRIC_ERR      acc [4][m] (+)= per column j [sum (b - a)^2 | sum |b - a| | sum (a - shift_j)
 *                                          | sum (a - shift_j)^2]; shift [m] float64 (device, nullable: 0); w unused
 *                      BKM_METRIC_LOGLOSS  a [n] int32 class index; b (n, m) probabilities, or m = 1: the probability
 *                                          of class 1 (then the row is [1 - b, b]).  q = clip(p, eps, 1 - eps),
 *                                          acc [2] (+)= [sum_i -w_i log(q_i[a_i] / sum_j q_ij) | sum_i w_i]; a class
 *                                          index outside the row makes the first sum NaN
 *                      OVERWRITTEN with BKM_FLAG_FIRST_CHUNK, else ACCUMULATED.  Threads add their rows in row order,
 *                      the row groups of a CTA and then the CTA partials are folded in a fixed order (no float
 *                      atomics): two calls with the same inputs give the same bits.  NaN operands propagate as in the
 *                      same float64 expression in numpy.  One launch.
 *                      workspace: bkm_metric_workspace_bytes(n, m, mode) bytes, any content. */
#define BKM_M_F16 3
#define BKM_M_I32 4
#define BKM_M_I64 5
#define BKM_M_U8  6   /* bool and uint8 */
#define BKM_METRIC_EQ      0
#define BKM_METRIC_ERR     1
#define BKM_METRIC_LOGLOSS 2
int bkm_metric_workspace_bytes(int64_t n, int m, int mode, size_t* out);
int bkm_metric_chunk(const void* a, int a_dtype, const void* b, int b_dtype, const double* w, int64_t n, int m,
                     int mode, const double* shift, double eps, double* acc, void* workspace, size_t ws_bytes,
                     int flags, void* stream);

/* ---- Per-column key tables: SimpleImputer's most-frequent counts and the encoders' categories ------------------------
 * A group of g columns owns keys / counts [total_slots] uint64, column j owning slots [slot_off[j], slot_off[j + 1])
 * (slot_off [g + 1] int64, device), a power of two (or zero).  Empty slots hold the key ~0 (a NaN pattern).  X + j0
 * with ldx runs a column group as a view.  Every value has an order-preserving 64-bit key: floats the radix key of
 * bkm_quantile_hist_chunk (16, 32 or 64 bits in a uint64) with -0.0 folded to +0.0 and every NaN mapped to the key of
 * the canonical quiet NaN (so NaN is one key, the largest); int32 / int64 the value with its sign bit flipped; uint8 the
 * value.  The tables are filled by bkm_mode_count_chunk (SimpleImputer) and bkm_distinct_chunk (the encoders); a
 * table's content is a set of keys with integer counts.
 *   bkm_mode_best        per column: best_key [g] uint64 and best_count [g] float64 of the entry of largest count, the
 *                        smallest key among equal counts (count 0: no value), and distinct [g] float64 the number of
 *                        occupied slots.  The order is total: the result does not depend on the table layout.  Several
 *                        CTAs share a column's table (slices, then a fold of their partials).  workspace:
 *                        bkm_mode_best_workspace_bytes(g, total_slots) bytes, any content.
 *   bkm_mode_compact     every occupied slot as a row of entries [*][4] float64 {column, key >> 32, key & 0xffffffff,
 *                        count}, rows in no particular order; *cursor (uint64, device) ends at the number of rows.
 *   bkm_mode_merge       resets the tables, then adds every row of entries [n_entries][4] with count > 0 to its
 *                        column's table (rows with count 0 are skipped: the zero padding of gathered slices). */
int bkm_mode_best_workspace_bytes(int g, int64_t total_slots, size_t* out);
int bkm_mode_best(const unsigned long long* keys, const unsigned long long* counts, const int64_t* slot_off, int g,
                  int64_t total_slots, unsigned long long* best_key, double* best_count, double* distinct,
                  void* workspace, size_t ws_bytes, void* stream);
int bkm_mode_compact(const unsigned long long* keys, const unsigned long long* counts, const int64_t* slot_off, int g,
                     double* entries, unsigned long long* cursor, void* stream);
int bkm_mode_merge(const double* entries, int64_t n_entries, unsigned long long* keys, unsigned long long* counts,
                   const int64_t* slot_off, int g, int64_t total_slots, void* stream);

/* ---- SimpleImputer: the fit statistics and the fill pass over row chunks (replace scikit-learn's _dense_fit, transform
 * and inverse_transform, which dask_ml/impute.py calls for numpy input) -------------------------------------------------
 * The missing value is passed as (miss_is_nan, miss_value): NaN when miss_is_nan = 1 (miss_value is then ignored, NaN
 * allowed), else every x with (double)x == miss_value (miss_value a value of X's dtype; +0.0 and -0.0 both match 0).
 *   bkm_impute_stats_chunk   acc [4][d] float64 per column: [missing count | NaN count | inf count | sum (x - shift_j)
 *                        over the non-missing finite x]; shift [d] float64 (device, nullable: 0).  OVERWRITTEN with
 *                        BKM_FLAG_FIRST_CHUNK, else ACCUMULATED; CTA partials are folded in a fixed order (no float
 *                        atomics): two calls with the same inputs give the same bits.  workspace:
 *                        bkm_impute_stats_workspace_bytes(n, d) bytes, any content.
 *   bkm_quantile_hist_masked_chunk   bkm_quantile_hist_chunk with the x == miss_value rows skipped as well (miss_value
 *                        not NaN), so that the select step's nvalid is the non-missing count.  Same state, rounds and
 *                        bkm_quantile_select_step.
 *   bkm_mode_count_chunk     per column j of a group of g columns, the count of every distinct non-missing, non-NaN
 *                        value, by its key, in the per-column key tables (above), each a power of two (or zero) at least
 *                        twice the values the column can receive, so that no table fills.  With BKM_FLAG_FIRST_CHUNK
 *                        the tables are reset first, else counts are ACCUMULATED.  Counts are integers: exact in any
 *                        order.  The best entry, compaction and multi-rank merge are bkm_mode_best / _compact / _merge.
 *   bkm_impute_chunk     forward (inverse 0): out [n][ld_out] in out_dtype (X's dtype; BKM_F32 for bf16 rows), columns
 *                        o < n_keep: x[:, cols[o]] with its missing elements replaced by (out_dtype)stats[cols[o]];
 *                        then n_ind indicator columns: 1 where x[:, cols[o]] is missing, else 0; then n_check input
 *                        columns cols[o] that are only validated.  invalid [2] float64 (nullable) (+)= the NaN and inf
 *                        counts of the filled and validated columns.  inverse (inverse 1): n_keep = n_ind = the output
 *                        width, cols [2 n_keep]: out[:, o] = x[:, cols[o]] (0 when cols[o] = -1), then miss_value where
 *                        x[:, cols[n_keep + o]] != 0 (cols[n_keep + o] >= 0).  One read of X, one write of out; any
 *                        ldx >= d, ld_out >= the output width; the input is only read. */
int bkm_impute_stats_workspace_bytes(int64_t n, int d, size_t* out);
int bkm_impute_stats_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int miss_is_nan, double miss_value,
                           const double* shift, double* acc, void* workspace, size_t ws_bytes, int flags, void* stream);
int bkm_quantile_hist_masked_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, double miss_value,
                                   const void* state, int n_q, int round, double* hist, int flags, void* stream);
int bkm_mode_count_chunk(const void* X, int64_t n, int g, int64_t ldx, int x_dtype, int miss_is_nan, double miss_value,
                         unsigned long long* keys, unsigned long long* counts, const int64_t* slot_off,
                         int64_t total_slots, int flags, void* stream);
int bkm_impute_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int miss_is_nan, double miss_value,
                     const double* stats, const int* cols, int n_keep, int n_ind, int n_check, int inverse, void* out,
                     int64_t ld_out, int out_dtype, double* invalid, void* stream);

/* ---- LabelEncoder / OneHotEncoder: the categories of every column and the encoding passes (replace da.unique,
 * np.searchsorted and the per-block sparse one-hot matrices of dask_ml/preprocessing/label.py and _encoders.py) --------
 * Element types of X: BKM_F32, BKM_F64, BKM_BF16, BKM_M_I32, BKM_M_I64, BKM_M_U8 (bool and uint8).  Values are
 * compared by their keys (the per-column key tables, above).
 *   bkm_distinct_chunk   per column j of a group of g columns, every distinct key, count 1, in the per-column key
 *                        tables (above); bkm_mode_compact, bkm_mode_merge and bkm_mode_best's distinct count read them.
 *                        state [2][g] uint64: [occupied slots | status bits]; status 1 = OVERFLOW (the occupancy passed
 *                        half the capacity or a probe chain passed 1024 slots: the column's table is incomplete, grow it
 *                        and run the group again), 2 = MARKER (the column holds the key ~0, i.e. INT64_MAX, which the
 *                        tables cannot store).  With BKM_FLAG_FIRST_CHUNK the tables and state are reset first, else
 *                        ACCUMULATED.
 *   bkm_encode_chunk     cat_keys [n_cats] uint64: column j's sorted keys at [cat_off[j], cat_off[j + 1]) (cat_off [d + 1]
 *                        int64, device).  The code of x[i, j] is the position of its key in its column's list.
 *                        layout CODES: out [n][ld_out >= d] int64 codes (-1 for an unknown key; out_dtype ignored).
 *                        layout DENSE: out [n][n_cats] (ld_out == n_cats, 16-byte aligned) in out_dtype (BKM_F64,
 *                        BKM_F32, BKM_M_I64, BKM_M_I32, BKM_M_U8): 1 at column cat_off[j] + code of every j, 0 elsewhere,
 *                        every element written once; d <= 2048.  layout CSR: indices [n d] int64 = cat_off[j] + code
 *                        (-1 for an unknown key) at i d + j, out [n d] ones in out_dtype.  unknown [1 + d + d
 *                        BKM_ENCODE_KEEP] uint64 (+)= [elements with an unknown key | per column: their count | per
 *                        column: up to BKM_ENCODE_KEEP of their keys, in no particular order]; the caller zeroes it.
 *   bkm_decode_chunk     codes [n][ldc] int32 / int64 (BKM_M_I32 / BKM_M_I64) -> out [n][ld_out] elements of elem_bytes
 *                        (1, 2, 4, 8): out[i, j] = cat_vals[cat_off[j] + codes[i, j]]; a code outside [0, K_j) writes
 *                        zero bytes and adds to unknown (as above, the code kept as the key). */
#define BKM_ENCODE_CODES 0
#define BKM_ENCODE_DENSE 1
#define BKM_ENCODE_CSR   2
#define BKM_ENCODE_KEEP  8
int bkm_distinct_chunk(const void* X, int64_t n, int g, int64_t ldx, int x_dtype, unsigned long long* keys,
                       unsigned long long* counts, const int64_t* slot_off, int64_t total_slots, unsigned long long* state,
                       int flags, void* stream);
int bkm_encode_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const unsigned long long* cat_keys,
                     const int64_t* cat_off, int64_t n_cats, int layout, void* out, int64_t ld_out, int out_dtype,
                     int64_t* indices, unsigned long long* unknown, void* stream);
int bkm_decode_chunk(const void* codes, int64_t n, int d, int64_t ldc, int code_dtype, const void* cat_vals,
                     const int64_t* cat_off, int elem_bytes, void* out, int64_t ld_out, unsigned long long* unknown,
                     void* stream);

/* ---- HashingVectorizer: the document-term matrix of one block of ASCII documents (replaces scikit-learn's
 * HashingVectorizer.transform, which dask_ml/feature_extraction/text.py maps over the blocks) --------------------------
 * buf [n_bytes] uint8 holds the documents back to back, document i at [doc_off[i], doc_off[i + 1]) (doc_off [n_docs + 1]
 * int64, device, doc_off[n_docs] = n_bytes), each ENDING in a byte that is not a word character (the caller appends one,
 * e.g. '\n'), so that no token spans two documents.  Word characters are [A-Za-z0-9_]; a token is a maximal run of two
 * or more of them (scikit-learn's default token_pattern on ASCII text), lowercased A-Z when `lowercase`; an n-gram is n
 * consecutive tokens of one document joined by one space, min_n <= n <= max_n (1 <= min_n).  An n-gram's hash h is
 * MurmurHash3 x86_32 with seed 0 over its bytes, as int32; its column is |h| % n_features (for h = -2^31:
 * (2^31 - 1 - (n_features - 1)) % n_features) and its sign -1 when alternate_sign and h < 0, else +1.  A row's value in
 * a column is the sum of the signs of its n-grams there, zeros kept (1 for every stored column when `binary`); with
 * norm BKM_TEXT_NORM_L1 / _L2 the row is divided by sum |v| / sqrt(sum v^2), accumulated in float64 (the squares rounded
 * to out_dtype first) and divided in float64 before the rounding to out_dtype, unless the sum is 0.  This is
 * scikit-learn 1.9's arithmetic (_hashing_fast.pyx, sum_duplicates, sparsefuncs_fast.pyx) bit for bit, for float32
 * while no value passes 2^24.
 *   bkm_text_workspace_bytes  workspace of the two calls below: (n_bytes, n_docs, 0) for bkm_text_tokens_chunk,
 *                        (n_bytes, n_docs, n_pairs) for bkm_text_hash_chunk; n_pairs <= INT_MAX.
 *   bkm_text_tokens_chunk  tok_start [tok_cap >= n_bytes / 3 + 1] int64 = the byte position of every token, ascending;
 *                        tok_off [n_docs + 1] int64 = each document's first token (tok_off[n_docs] = the token count);
 *                        pair_off [n_docs + 1] int64 = each document's first n-gram (the exclusive scan of the n-gram
 *                        counts); totals[0] = tokens, totals[1] = n-grams (int64, device).
 *   bkm_text_hash_chunk  keys [n_pairs] uint32 = 2 column + (1 for sign -1) of every n-gram, sorted within each
 *                        document; indptr [n_docs + 1] int64 = the CSR row offsets; scale [n_docs] float64 = each row's
 *                        divisor (0: not divided); totals[2] = stored entries.  n_tokens, n_pairs: totals[0], totals[1].
 *   bkm_text_write_chunk indices [totals[2]] int64, ascending within a row, and data [totals[2]] in out_dtype (BKM_F32 or
 *                        BKM_F64) of every stored entry. */
#define BKM_TEXT_NORM_NONE 0
#define BKM_TEXT_NORM_L1   1
#define BKM_TEXT_NORM_L2   2
int bkm_text_workspace_bytes(int64_t n_bytes, int64_t n_docs, int64_t n_pairs, size_t* out);
int bkm_text_tokens_chunk(const uint8_t* buf, int64_t n_bytes, const int64_t* doc_off, int64_t n_docs, int min_n,
                          int max_n, int64_t* tok_start, int64_t tok_cap, int64_t* tok_off, int64_t* pair_off,
                          int64_t* totals, void* workspace, size_t ws_bytes, void* stream);
int bkm_text_hash_chunk(const uint8_t* buf, int64_t n_bytes, const int64_t* tok_start, const int64_t* tok_off,
                        const int64_t* pair_off, int64_t n_docs, int64_t n_tokens, int64_t n_pairs, int min_n, int max_n,
                        int lowercase, int64_t n_features, int alternate_sign, int binary, int norm, int out_dtype,
                        uint32_t* keys, int64_t* indptr, double* scale, int64_t* totals, void* workspace,
                        size_t ws_bytes, void* stream);
int bkm_text_write_chunk(const uint32_t* keys, const int64_t* pair_off, const int64_t* indptr, const double* scale,
                         int64_t n_docs, int binary, int64_t* indices, void* data, int out_dtype, void* stream);

/* ---- one epoch of scikit-learn's _plain_sgd over one block, for P independent binary problems --------------------
 *   bkm_sgd_order      HOST function, no CUDA: out_host[0..n) = the row order of SequentialDataset.shuffle(seed) (the
 *                      Fisher-Yates shuffle driven by our_rand_r, sklearn/utils/_random.pxd), n <= 2^31 - 1.
 *   bkm_sgd_block      rows of a dense block X (n, d), any row pitch ldx, float32 or float64.
 *   bkm_sgd_csr_block  rows of a CSR block (crow int64 (n + 1), col int64 (nnz), val float32 / float64 (nnz)) of d
 *                      columns; each row's entries are visited in stored order, as CSRDataset does.
 * Problem p (0 <= p < P) visits the rows order[p*n + 0 .. n) (int32) with the labels y[p*n + row] (float64, in the
 * block's row order) and sample_weight[row] (float64, NULL = 1) and updates, in float64:
 *   w    (P, d)  the weights (WeightVector.w with wscale = 1 on entry and exit)
 *   aw   (P, d)  the average weights, NULL without `average`
 *   q    (P, d)  scratch of the L1 / elasticnet penalty (zeroed by the call), NULL otherwise
 *   st   (P, 4)  [intercept | average intercept | non-finite flag | unused]: the flag is set to 1 when an intercept or
 *                weight is not finite after the epoch (scikit-learn's under/overflow ValueError); w is then left
 *                unscaled, as scikit-learn raises before reset_wscale.
 *   cw   (P, 2)  [weight_pos | weight_neg] per problem.
 * `eta` (n, float64) is the per-step learning rate of 'invscaling' (eta0 / pow(t, power_t), computed on the host),
 * NULL otherwise.  Every product and sum is rounded on its own, in the order of _plain_sgd and WeightVector, except the
 * fold of w into aw in reset_wscale, which is fused as the x86-64 BLAS daxpy fuses it; so everything but the exp of
 * log_loss matches scikit-learn's float64 path bit for bit.  One launch; a CTA per
 * problem.  w, aw and q stay in shared memory for the epoch when 8 d (1 + [aw] + [q]) bytes fit, in global memory
 * otherwise. */
#define BKM_SGD_HINGE 0                 /* threshold = epsilon (1 for hinge, 0 for perceptron) */
#define BKM_SGD_LOG 1
#define BKM_SGD_MODIFIED_HUBER 2
#define BKM_SGD_SQUARED_HINGE 3         /* threshold = epsilon */
#define BKM_SGD_SQUARED_ERROR 4
#define BKM_SGD_HUBER 5
#define BKM_SGD_EPS_INSENSITIVE 6
#define BKM_SGD_SQ_EPS_INSENSITIVE 7
typedef struct {
  int loss, penalty, learning_rate, fit_intercept;   /* penalty 0 none, 1 l1, 2 l2, 3 elasticnet; learning_rate as
                                                        _sgd_fast: 1 constant, 2 optimal, 3 invscaling, 4 adaptive,
                                                        5 pa1, 6 pa2 */
  double epsilon, alpha, l1_ratio, eta0, optimal_init, t0, intercept_decay, average;
} bkm_sgd_params;
int bkm_sgd_order(int64_t n, uint32_t seed, int32_t* out_host);
int bkm_sgd_block(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* order, const double* y,
                  const double* sample_weight, const double* eta, const double* cw, int P,
                  const bkm_sgd_params* params_host, double* w, double* aw, double* q, double* st, void* stream);
int bkm_sgd_csr_block(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n, int d,
                      int64_t nnz, const int32_t* order, const double* y, const double* sample_weight,
                      const double* eta, const double* cw, int P, const bkm_sgd_params* params_host, double* w,
                      double* aw, double* q, double* st, void* stream);

/* ---- NaN/inf scan of a chunk (k_means.py:179-180): sets *flag (int32) nonzero -------- */
int bkm_check_finite(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                     int* flag, void* stream);

/* ---- the per-iteration collective over NVLink peer memory (N > 1 GPUs of one node) --------------------------------
 * Replaces the `da.atop(..., sum)` / bincount fold across workers (k_means.py:545-550), i.e. the all-reduce of
 * [k*d sums | k counts | inertia].  Every rank owns a MAILBOX (bkm_p2p_mailbox_bytes / bkm_p2p_alloc: one cudaMalloc
 * allocation, zeroed), exports it (64-byte IPC handle), opens every peer's (bkm_p2p_import) and passes the device array
 * of the `world` mailbox pointers to bkm_allreduce_p2p: one kernel pushes `buf` into a slot of every mailbox, raises a
 * flag, waits for all flags in its own mailbox (2 s wall-clock limit: a timeout poisons buf[0] with NaN) and adds the slots
 * in RANK order — every rank ends with bit-identical sums.  `seq` = 1, 2, 3, ... the call number, identical on all ranks;
 * n <= max_elems (the slot size the mailboxes were sized for). */
int bkm_p2p_mailbox_bytes(int world, int64_t max_elems, size_t* nbytes);
int bkm_p2p_alloc(size_t nbytes, void** dev_ptr);
int bkm_p2p_free(void* dev_ptr);
int bkm_p2p_export(void* dev_ptr, void* handle64_host);
int bkm_p2p_import(const void* handle64_host, void** dev_ptr);
int bkm_p2p_close(void* dev_ptr);
int bkm_allreduce_p2p(double* buf, int64_t n, void* const* mailboxes_dev, int rank, int world, int64_t max_elems,
                      unsigned int seq, void* stream);

/* Number of kernel launches this library has enqueued since load (for bench accounting). */
int64_t bkm_launch_count(void);
/* Number of chunk calls whose shape belongs to the tensor-core / streaming family but whose rows were not 16-byte aligned
 * (base or pitch), so that the generic CUDA-core kernel ran instead: correct, several times slower.  The Python host
 * warns once when this moves. */
int64_t bkm_debug_fallback_count(void);

/* Debug: nonzero once a pipeline wait inside a tensor-core kernel has timed out (the kernel then drains
 * instead of hanging); encodes barrier / parity / warp.  Synchronises the device. */
unsigned int bkm_debug_abort_code(void);
void bkm_debug_abort_detail(unsigned int* out64_host);   /* per-warp wait that timed out (64 words) */
/* Clears the abort word once the host has reported it (the host side raises RuntimeError on a non-finite shift /
 * cost and calls this, so that one timed-out wait does not poison the process).  Synchronises the device. */
void bkm_debug_reset(void);
/* Number of rows the LAST tensor-core chunk call that used `workspace` (same n, d, k, dtype) deferred to the float64
 * re-check (near-ties and out-of-range rows).  Synchronises the device; used by bench.py's parity record. */
int bkm_debug_deferred_rows(const void* workspace, int64_t n, int d, int k, int x_dtype, int* count_host);
/* Pipeline timeline of the tensor-core kernel: not recorded by the sm_90a kernels; returns 0 (kept for ABI stability) */
int bkm_debug_trace(long long* out_host, int n);

#ifdef __cplusplus
}
#endif
#endif /* BKM_B200_H */

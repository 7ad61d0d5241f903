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

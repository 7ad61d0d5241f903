// bkm_api.cu — the extern "C" boundary declared in include/bkm_b200.h: argument validation,
// kernel-family dispatch, workspace carving.  No allocation, no synchronisation, no throws.
#include "bkm_common.cuh"
#include <math.h>

namespace bkm {
unsigned int tc_abort_code();
void tc_abort_detail(unsigned int* out64);
void tc_abort_reset();
int launch_pack(const double* C, int k, int d, int dtype, void* pack, cudaStream_t s);
int launch_make_blobs(void* X, long long* y, long long n, int d, long long ldx, int dtype, const double* centers,
                      const double* stds, int k, uint64_t seed, int sm_count, cudaStream_t s);
int launch_min_fold(void* run_min, const void* new_min, long long n, int dtype, double* phi_acc, int sm_count, cudaStream_t s);
int launch_loop_reset(void* state, double tol, double* hist, int hist_cap, cudaStream_t s);
int launch_finalize_step(const double* red, const double* c_in, double* c_out, void* state, int k, int d, int dtype,
                         void* pack, cudaStream_t s);
int launch_minibatch_step(const double* red, const double* c_in, const double* w_in, double* c_out, double* w_out,
                          int k, int d, int dtype, void* pack, cudaStream_t s);
int launch_finalize(const double* sums, const long long* counts, const double* Cold, double* Cnew,
                    double* shift, int k, int d, cudaStream_t s);
int launch_sample(const void* d2, long long n, int dtype, double eop, uint64_t seed, uint64_t off,
                  long long* picked, long long cap, int* n_picked, cudaStream_t s);
int launch_transform(const void* X, long long n, int d, long long ldx, int dtype,
                     const void* pack, int k, void* out, long long ld_out, int mode, double gamma, int sm_count,
                     cudaStream_t s);
int launch_check_finite(const void* X, long long n, int d, long long ldx, int dtype, int* flag,
                        int sm_count, cudaStream_t s);
int launch_nystrom(const void* X, long long n, int d, long long ldx, int dtype, const void* pack, int l, double gamma,
                   int mode, const void* W, int kw, void* out, long long ld_out, double* part, size_t part_bytes,
                   int sm_count, int* parts_out, cudaStream_t s);
int launch_colsum_fold(const double* part, int parts, int l, double* colsum, int first, cudaStream_t s);

static std::atomic<int> g_sm_count[64];
int sm_count(int* out) {
  int dev = 0;
  BKM_CUDA_TRY(cudaGetDevice(&dev));
  if (dev < 0 || dev >= 64) return BKM_EINVAL;
  int v = g_sm_count[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    BKM_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
    g_sm_count[dev].store(v, std::memory_order_relaxed);
  }
  *out = v;
  return 0;
}

static std::atomic<long long> g_fallbacks{0};   // chunk calls that left their shape's kernel family for the generic kernel

// Near-tie margin coefficient: a row is re-evaluated in float64 when
//   second_best - best <= tau * (||x||^2 + max_j ||c_j||^2).
// fp32 dot products of length d carry a rounding error of about sqrt(d)*2^-24 relative to
// sum|x_i c_i| <= (||x||^2+||c||^2)/2; both distances and the -2 factor give the constant.
static float tau_for(int d, int dtype, int flags, int family) {
  if (dtype == BKM_F64 || (flags & BKM_FLAG_NO_RECHECK)) return 0.f;
  const float eps = 1.0f / 16777216.0f;   // 2^-24
  // large-shape tensor path: bf16 rows are exact operands; the centres are a bf16 (hi, lo) pair: |c - hi - lo| <= 2^-18 |c|,
  // so |sum x_i r_i| <= 2^-19 (||x||^2 + ||c||^2), doubled by the -2 factor and again for the difference of two
  // distances: 2^-17.  To that the fp32 accumulation of 2 products per 16-element K-step (same model as family 1).
  if (family == 3) return 1.0f / 131072.0f + (8.0f * sqrtf(2.0f * (float)((d + 7) / 8)) + 16.0f) * eps;
  // tensor path (split-fp16 triple, scaled by a power of two): error sources relative to ||x||^2+||c||^2 are the
  // fp16 (hi, lo) representation of both operands (2^-22 each; 2^-25 absolute in scaled units when lo falls into
  // fp16's subnormals, negligible because the scale puts max|c| at 2^9..2^10), the dropped lo*lo term (2^-24),
  // the 3*ceil(d/16) accumulations into the fp32 accumulator, the fp32 addition of ||s c||^2, and the accumulator's own
  // rounding.  tests/test_gpu_tau.py measures, with the re-check switched off, the worst margin of a label that differs
  // from float64 and asserts at least 4x headroom to this bound (3.3e-6 at d=64); the parity tests assert that every
  // remaining difference is a float64 near-tie (<= 1e-9).
  if (family == 1) return (8.0f * sqrtf(3.0f * (float)((d + 7) / 8)) + 16.0f) * eps;
  // CUDA-core kernels (generic and streaming): fp32 FMA chains of length d plus the rounding of ||c||^2
  return 8.0f * (sqrtf((float)d) + 2.0f) * eps;
}

static int chunk_common(const void* X, long long n, int d, long long ldx, int x_dtype,
                        const void* pack, int k, int* labels, void* min_out, int squared,
                        bool mstep, double* sums, long long* counts, double* dist_sum,
                        void* ws, size_t ws_bytes, int flags, const void* loop_state, cudaStream_t s) {
  if (n < 0 || d <= 0 || k <= 0 || ldx < d) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (!pack || !ws) return BKM_EINVAL;
  if (mstep && (!sums || !counts)) return BKM_EINVAL;
  if (n == 0) return 0;
  if (!X) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  WsLayout W = ws_layout(n, d, k, x_dtype, sm);
  if (ws_bytes < W.total) return BKM_EWORKSPACE;
  if (n > 0x7fffffffLL) return BKM_EUNSUPPORTED;      // row indices inside a chunk are 32-bit

  ChunkArgs a;
  a.X = X; a.n = n; a.d = d; a.ldx = ldx;
  a.pack = (const unsigned char*)pack;
  a.L = pack_layout(k, d, x_dtype);
  a.k = k; a.labels = labels; a.min_out = min_out; a.squared = squared;
  a.psum = (unsigned char*)ws + W.off_psum;
  a.pcnt = (int*)((unsigned char*)ws + W.off_pcnt);
  a.pin = (double*)((unsigned char*)ws + W.off_pin);
  a.want_sum = dist_sum != nullptr;
  a.psum_slots = W.psum_slots;
  a.part_slots = W.part_slots;
  a.defer_cnt = (int*)((unsigned char*)ws + W.off_flag);
  a.defer_idx = (int*)((unsigned char*)ws + W.off_defer);
  a.out_sums = sums; a.out_counts = counts; a.out_dist_sum = dist_sum;
  a.skip = loop_state ? &reinterpret_cast<const LoopState*>(loop_state)->done : nullptr;
  a.first_chunk = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  a.counts_f64 = (flags & BKM_FLAG_COUNTS_F64) ? 1 : 0;
  a.rec = reinterpret_cast<float4*>((unsigned char*)ws + W.off_rec);
  a.bin_list = (unsigned char*)ws + W.off_bin;
  a.bin_off = (int*)((unsigned char*)ws + W.off_binoff);
  a.bal = (unsigned char*)ws + W.off_bal;

  int family = bkm_kernel_family(d, k, x_dtype, flags);
  if (family < 0) return family;
  a.tau = tau_for(d, x_dtype, flags, family);
  int grid = 0;
  rc = BKM_EALIGN;
  if (family == 3) {
    // large-shape tensor path: E-step kernel (+ slice combine + float64 re-check), then label-indexed row passes
    if (!a.labels) a.labels = (int*)((unsigned char*)ws + W.off_lab);
    int parts = 0;
    rc = launch_tc2(a, mstep, sm, &parts, s);
    if (rc) return rc;                                  // bf16 rows have no CUDA-core fallback (BKM_EALIGN: 16-byte rows)
    const int mparts = parts & 0xffff, dparts = parts >> 16;
    return launch_reduce_partials(a, mparts, mparts, dparts, mstep, x_dtype, sums, counts, dist_sum, s);
  }
  if (family == 1) {
    rc = launch_tc(a, mstep, sm, &grid, s);
    if (rc == BKM_EALIGN && !(flags & BKM_FLAG_FORCE_TC)) {   // TMA needs 16-byte aligned rows
      g_fallbacks.fetch_add(1, std::memory_order_relaxed);
      family = 0;
      a.tau = tau_for(d, x_dtype, flags, 0);
    }
  }
  if (family == 2) {
    rc = launch_stream(a, mstep, sm, &grid, s);
    if (rc == BKM_EALIGN || rc == BKM_EUNSUPPORTED) {          // odd base pointer / very wide pitch: generic kernel
      g_fallbacks.fetch_add(1, std::memory_order_relaxed);
      family = 0;
      a.tau = tau_for(d, x_dtype, flags, 0);
    }
  }
  if (family == 0) rc = launch_simt(a, mstep, x_dtype, sm, &grid, s);
  if (rc) return rc;
  // grid < 0: the generic kernel ran in GLOBAL mode (sums accumulated by float64 atomics into slot 0)
  const int g = grid < 0 ? -grid : grid;
  rc = launch_reduce_partials(a, grid < 0 ? 1 : g, g, g, mstep, grid < 0 ? BKM_F64 : x_dtype, sums, counts, dist_sum, s);
  if (rc) return rc;
  if (family == 1) rc = launch_tc_recheck(a, mstep, sm, s);     // float64 decisions of the deferred rows, added on top
  return rc;
}

}  // namespace bkm

using namespace bkm;

extern "C" {

int bkm_version(void) { return BKM_VERSION; }

const char* bkm_error_string(int code) {
  switch (code) {
    case BKM_OK: return "ok";
    case BKM_EINVAL: return "invalid argument";
    case BKM_EDTYPE: return "unsupported dtype";
    case BKM_EUNSUPPORTED: return "shape not supported by any kernel";
    case BKM_EWORKSPACE: return "workspace too small";
    case BKM_EALIGN: return "pointer alignment";
    default: break;
  }
  if (code > 0) return cudaGetErrorString((cudaError_t)code);
  return "unknown error";
}

int bkm_device_info(int device, int* sm_count, int* cc_major, int* cc_minor) {
  int v = 0;
  BKM_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device));
  if (sm_count) *sm_count = v;
  BKM_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMajor, device));
  if (cc_major) *cc_major = v;
  BKM_CUDA_TRY(cudaDeviceGetAttribute(&v, cudaDevAttrComputeCapabilityMinor, device));
  if (cc_minor) *cc_minor = v;
  return 0;
}

int bkm_kernel_family(int d, int k, int x_dtype, int flags) {
  if (d <= 0 || k <= 0) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (x_dtype == BKM_BF16) return tc2_shape(d, k, x_dtype) ? 3 : BKM_EUNSUPPORTED;     // bf16 rows: tensor path only
  bool tc = tc_supported(d, k, x_dtype);
  if (flags & BKM_FLAG_FORCE_SIMT) return 0;
  if (flags & BKM_FLAG_FORCE_TC) return tc ? 1 : BKM_EUNSUPPORTED;
  // The tensor kernel costs ~20 ns per row and SM whatever k and d are (per-tile pipeline costs): tiny problems
  // (C4: d=13, k=20) are HBM-bound and go to the streaming CUDA-core kernel (family 2, bkm_stream.cu).
  if (stream_supported(d, k, x_dtype) && (long long)k * d < 512) return 2;
  return (tc && (long long)k * d >= 512) ? 1 : 0;
}

int bkm_centers_pack_bytes(int k, int d, int x_dtype, size_t* out) {
  if (k <= 0 || d <= 0 || !out) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  *out = pack_layout(k, d, x_dtype).total;
  return 0;
}

int bkm_pack_centers(const double* centers64, int k, int d, int x_dtype, void* pack,
                     size_t pack_bytes, void* stream) {
  if (!centers64 || !pack || k <= 0 || d <= 0) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (pack_bytes < pack_layout(k, d, x_dtype).total) return BKM_EWORKSPACE;
  if ((uintptr_t)pack & 255) return BKM_EALIGN;
  return launch_pack(centers64, k, d, x_dtype, pack, (cudaStream_t)stream);
}

int bkm_workspace_bytes(int64_t n, int d, int k, int x_dtype, size_t* out) {
  if (k <= 0 || d <= 0 || n < 0 || !out) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  *out = ws_layout(n, d, k, x_dtype, sm_count_or_default()).total;
  return 0;
}

int bkm_lloyd_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack,
                    int k, int32_t* labels, void* min_d2, double* sums, int64_t* counts,
                    double* inertia, void* workspace, size_t workspace_bytes, int flags,
                    const void* loop_state, void* stream) {
  return chunk_common(X, n, d, ldx, x_dtype, pack, k, labels, min_d2, 1, true, sums,
                      (long long*)counts, inertia, workspace, workspace_bytes, flags, loop_state,
                      (cudaStream_t)stream);
}

int bkm_assign_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack,
                     int k, int32_t* labels, void* min_dist, int squared, double* dist_sum,
                     void* workspace, size_t workspace_bytes, int flags, void* stream) {
  return chunk_common(X, n, d, ldx, x_dtype, pack, k, labels, min_dist, squared ? 1 : 0, false,
                      nullptr, nullptr, dist_sum, workspace, workspace_bytes, flags, nullptr,
                      (cudaStream_t)stream);
}

int bkm_sample_chunk(const void* min_d2, int64_t n, int x_dtype, double ell_over_phi,
                     uint64_t seed, uint64_t row_offset, int64_t* picked, int64_t cap,
                     int* n_picked, void* stream) {
  if (n < 0 || cap < 0 || !n_picked || (cap > 0 && !picked)) return BKM_EINVAL;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n > 0 && !min_d2) return BKM_EINVAL;
  return launch_sample(min_d2, n, x_dtype, ell_over_phi, seed, row_offset, (long long*)picked, cap,
                       n_picked, (cudaStream_t)stream);
}

int bkm_transform_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype,
                        const void* pack, int k, void* out, int64_t ld_out, int mode, double gamma, int flags,
                        void* stream) {
  if (n < 0 || d <= 0 || k <= 0 || ldx < d || !pack || ld_out < k || mode < 0 || mode > 2) return BKM_EINVAL;
  if (n > 0x7fffffffLL) return BKM_EUNSUPPORTED;      // TMA row coordinates of the tensor path are 32-bit
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X || !out) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  // fp32, d <= 64, k <= 256: the tensor-core kernel with the transform epilogue (callers cut wider Y into column blocks)
  if (x_dtype == BKM_F32 && tc_supported(d, k, x_dtype) && !(flags & BKM_FLAG_FORCE_SIMT)) {
    ChunkArgs a = {};
    a.X = X; a.n = n; a.d = d; a.ldx = ldx;
    a.pack = (const unsigned char*)pack;
    a.L = pack_layout(k, d, x_dtype);
    a.k = k;
    a.xf_out = (float*)out; a.xf_ld = ld_out; a.xf_mode = mode; a.xf_gamma = gamma;
    rc = launch_tc_transform(a, sm, (cudaStream_t)stream);
    if (rc != BKM_EALIGN && rc != BKM_EUNSUPPORTED) return rc;
    if (flags & BKM_FLAG_FORCE_TC) return rc;
    if (rc == BKM_EALIGN) g_fallbacks.fetch_add(1, std::memory_order_relaxed);
  } else if (flags & BKM_FLAG_FORCE_TC) return BKM_EUNSUPPORTED;
  return launch_transform(X, n, d, ldx, x_dtype, pack, k, out, ld_out, mode, gamma, sm, (cudaStream_t)stream);
}

// Nystrom passes (spectral.py:237-270): fp32 rows with d <= 64, l <= 256 (and k <= 64 outputs) run on the tensor-core
// kernel's COLSUM / EMBED epilogues; every other shape, float64 rows and unaligned fp32 rows on the CUDA-core kernel
static ChunkArgs nystrom_args(const void* X, int64_t n, int d, int64_t ldx, const void* pack, int l, double gamma) {
  ChunkArgs a = {};
  a.X = X; a.n = n; a.d = d; a.ldx = ldx;
  a.pack = (const unsigned char*)pack;
  a.L = pack_layout(l, d, BKM_F32);
  a.k = l;
  a.xf_gamma = gamma;
  return a;
}

int bkm_kernel_colsum_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack, int l,
                            double gamma, double* colsum, void* workspace, size_t workspace_bytes, int flags,
                            void* stream) {
  if (n < 0 || d <= 0 || l <= 0 || ldx < d || !pack || !colsum || !workspace) return BKM_EINVAL;
  if (n > 0x7fffffffLL) return BKM_EUNSUPPORTED;      // TMA row coordinates of the tensor path are 32-bit
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n > 0 && !X) return BKM_EINVAL;
  cudaStream_t s = (cudaStream_t)stream;
  const int first = (flags & BKM_FLAG_FIRST_CHUNK) ? 1 : 0;
  if (n == 0) {
    if (first) BKM_CUDA_TRY(cudaMemsetAsync(colsum, 0, (size_t)l * sizeof(double), s));
    return 0;
  }
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  // The per-CTA partials go behind the workspace's persistent header (WsLayout::off_bal is left alone), into the
  // per-call area of a chunk call with k = l: it holds at least the counts region, part_slots x l int32 = 4 x SMs
  // slots of l float64, the most either kernel writes (tensor path: 2 per CTA, one CTA per SM; CUDA cores: <= 4 x SMs
  // CTAs); launch_tc_colsum / launch_nystrom check the size they need against it.
  const WsLayout WL = ws_layout(n, d, l, x_dtype, sm);
  if (workspace_bytes < WL.total) return BKM_EWORKSPACE;
  double* part = (double*)((unsigned char*)workspace + WL.off_psum);
  const size_t part_bytes = workspace_bytes - WL.off_psum;
  int parts = 0;
  rc = BKM_EALIGN;
  if (x_dtype == BKM_F32 && tc_supported(d, l, x_dtype) && !(flags & BKM_FLAG_FORCE_SIMT)) {
    rc = launch_tc_colsum(nystrom_args(X, n, d, ldx, pack, l, gamma), part, part_bytes, sm, &parts, s);
    if (rc != 0 && (flags & BKM_FLAG_FORCE_TC)) return rc;
    if (rc != 0 && rc != BKM_EALIGN) return rc;
    if (rc == BKM_EALIGN) g_fallbacks.fetch_add(1, std::memory_order_relaxed);
  } else if (flags & BKM_FLAG_FORCE_TC) return BKM_EUNSUPPORTED;
  if (rc != 0) {
    rc = launch_nystrom(X, n, d, ldx, x_dtype, pack, l, gamma, 0, nullptr, 0, nullptr, 0, part, part_bytes, sm, &parts, s);
    if (rc) return rc;
  }
  return launch_colsum_fold(part, parts, l, colsum, first, s);
}

int bkm_nystrom_embed_chunk(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const void* pack, int l,
                            double gamma, const void* W, int k, void* out, int64_t ld_out, int flags, void* stream) {
  if (n < 0 || d <= 0 || l <= 0 || k <= 0 || ldx < d || ld_out < k || !pack || !W) return BKM_EINVAL;
  if (n > 0x7fffffffLL) return BKM_EUNSUPPORTED;      // TMA row coordinates of the tensor path are 32-bit
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X || !out) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (x_dtype == BKM_F32 && tc_supported(d, l, x_dtype) && k <= 64 && !(flags & BKM_FLAG_FORCE_SIMT)) {
    ChunkArgs a = nystrom_args(X, n, d, ldx, pack, l, gamma);
    a.xf_out = (float*)out; a.xf_ld = ld_out;
    rc = launch_tc_embed(a, (const float*)W, k, sm, s);
    if (rc != BKM_EALIGN || (flags & BKM_FLAG_FORCE_TC)) return rc;
    g_fallbacks.fetch_add(1, std::memory_order_relaxed);
  } else if (flags & BKM_FLAG_FORCE_TC) return BKM_EUNSUPPORTED;
  int parts = 0;
  return launch_nystrom(X, n, d, ldx, x_dtype, pack, l, gamma, 1, W, k, out, ld_out, nullptr, 0, sm, &parts, s);
}

int bkm_finalize(const double* sums, const int64_t* counts, const double* centers_old,
                 double* centers_new, double* shift, int k, int d, void* stream) {
  if (!sums || !counts || !centers_old || !centers_new || !shift || k <= 0 || d <= 0) return BKM_EINVAL;
  return launch_finalize(sums, (const long long*)counts, centers_old, centers_new, shift, k, d,
                         (cudaStream_t)stream);
}

int bkm_min_fold_chunk(void* run_min, const void* new_min, int64_t n, int x_dtype, double* phi_acc, void* stream) {
  if (n < 0) return BKM_EINVAL;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!run_min) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  return launch_min_fold(run_min, new_min, n, x_dtype, phi_acc, sm, (cudaStream_t)stream);
}

int bkm_make_blobs_chunk(void* X, int64_t* y, int64_t n, int d, int64_t ldx, int x_dtype, const double* centers,
                         const double* cluster_std, int k, uint64_t seed, void* stream) {
  if (n < 0 || d <= 0 || k <= 0 || ldx < d || !centers || !cluster_std) return BKM_EINVAL;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  return launch_make_blobs(X, (long long*)y, n, d, ldx, x_dtype, centers, cluster_std, k, seed, sm, (cudaStream_t)stream);
}

int bkm_loop_state_bytes(size_t* out) {
  if (!out) return BKM_EINVAL;
  *out = sizeof(LoopState);
  return 0;
}

int bkm_loop_reset(void* loop_state, double tol, double* shift_hist, int hist_cap, void* stream) {
  if (!loop_state || hist_cap < 0 || (hist_cap > 0 && !shift_hist)) return BKM_EINVAL;
  if ((uintptr_t)loop_state & 7) return BKM_EALIGN;
  return launch_loop_reset(loop_state, tol, shift_hist, hist_cap, (cudaStream_t)stream);
}

int bkm_finalize_step(const double* reduced, const double* centers_in, double* centers_out, void* loop_state,
                      int k, int d, int x_dtype, void* pack, size_t pack_bytes, void* stream) {
  if (!reduced || !centers_in || !centers_out || !loop_state || !pack || k <= 0 || d <= 0) return BKM_EINVAL;
  if (centers_in == centers_out) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (pack_bytes < pack_layout(k, d, x_dtype).total) return BKM_EWORKSPACE;
  if (((uintptr_t)pack & 255) || ((uintptr_t)loop_state & 7)) return BKM_EALIGN;
  return launch_finalize_step(reduced, centers_in, centers_out, loop_state, k, d, x_dtype, pack, (cudaStream_t)stream);
}

int bkm_minibatch_step(const double* reduced, const double* centers_in, const double* weights_in, double* centers_out,
                       double* weights_out, int k, int d, int x_dtype, void* pack, size_t pack_bytes, void* stream) {
  if (!reduced || !centers_in || !weights_in || !centers_out || !weights_out || !pack || k <= 0 || d <= 0)
    return BKM_EINVAL;
  if (centers_in == centers_out || weights_in == weights_out) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (pack_bytes < pack_layout(k, d, x_dtype).total) return BKM_EWORKSPACE;
  if ((uintptr_t)pack & 255) return BKM_EALIGN;
  return launch_minibatch_step(reduced, centers_in, weights_in, centers_out, weights_out, k, d, x_dtype, pack,
                               (cudaStream_t)stream);
}

int bkm_check_finite(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, int* flag,
                     void* stream) {
  if (n < 0 || d <= 0 || ldx < d || !flag) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  if (n == 0) return 0;
  if (!X) return BKM_EINVAL;
  int sm = 0;
  int rc = sm_count(&sm);
  if (rc) return rc;
  return launch_check_finite(X, n, d, ldx, x_dtype, flag, sm, (cudaStream_t)stream);
}

int64_t bkm_launch_count(void) { return (int64_t)g_launches.load(); }
int64_t bkm_debug_fallback_count(void) { return (int64_t)g_fallbacks.load(); }

unsigned int bkm_debug_abort_code(void) { return bkm::tc_abort_code(); }
void bkm_debug_abort_detail(unsigned int* out64_host) { bkm::tc_abort_detail(out64_host); }
void bkm_debug_reset(void) { bkm::tc_abort_reset(); }

int bkm_debug_deferred_rows(const void* workspace, int64_t n, int d, int k, int x_dtype, int* count_host) {
  if (!workspace || !count_host || n < 0 || d <= 0 || k <= 0) return BKM_EINVAL;
  if (!dtype_ok(x_dtype)) return BKM_EDTYPE;
  WsLayout W = ws_layout(n, d, k, x_dtype, sm_count_or_default());
  BKM_CUDA_TRY(cudaMemcpy(count_host, (const unsigned char*)workspace + W.off_flag, sizeof(int), cudaMemcpyDeviceToHost));
  return 0;
}
int bkm_debug_trace(long long* out_host, int n) { return bkm::tc_trace(out_host, n); }

// The CUDA-core kernel a chunk call would run, with chunk_common's fallbacks, from the configuration functions its
// launches use (host only, no device call)
int bkm_debug_core_layout(int d, int k, int64_t ldx, int x_dtype, int flags, int mstep, int aligned16, int* out) {
  if (!out || d <= 0 || k <= 0 || ldx < d) return BKM_EINVAL;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return dtype_ok(x_dtype) ? BKM_EUNSUPPORTED : BKM_EDTYPE;
  int family = bkm_kernel_family(d, k, x_dtype, flags);
  if (family < 0) return family;
  // the tensor-core kernel runs unless the rows are not 16-byte aligned (and FORCE_TC does not forbid the fallback)
  if (family == 1 && ((aligned16 && ldx % 4 == 0) || (flags & BKM_FLAG_FORCE_TC))) return BKM_EUNSUPPORTED;
  for (int i = 0; i < 13; ++i) out[i] = 0;
  if (family == 2 && aligned16 && stream_layout(d, k, ldx, out) == 0) return 0;
  for (int i = 0; i < 13; ++i) out[i] = 0;
  return simt_layout(d, k, x_dtype, mstep != 0, out);
}

}  // extern "C"

// bkm_sgd.cu — one epoch of scikit-learn's _plain_sgd (sklearn/linear_model/_sgd_fast.pyx.tp) over one row block, for
// P independent binary problems (sm_90a).  Built with -fmad=false: every product and sum is rounded on its own.
//
//   bkm_sgd_order      the row order of SequentialDataset.shuffle(seed), on the host.
//   bkm_sgd_block      dense rows (float32 / float64, any row pitch).
//   bkm_sgd_csr_block  the rows of a CSR block, each row's entries in stored order.
//
// One CTA per problem walks that problem's rows in its order.  Per row:
//   1. the row's entries are staged in shared memory, kTile at a time: every thread stages x_j and forms the products
//      w[idx] * x_j (and, for PA, x_j * x_j) of its entries, each rounded on its own; thread 0 then only adds the staged
//      products in stored order: one summation chain per dot product, as WeightVector.dot and sqnorm do;
//   2. thread 0 runs the scalar part of the step (prediction, learning rate, loss gradient, clipping, class and sample
//      weight, w.scale, intercept, averaging and L1 scalars) exactly as _plain_sgd orders it;
//   3. all threads apply the per-entry updates (w.add, w.add_average, l1penalty), each entry owned by one thread, after
//      the rare reset_wscale of w.scale has run over the whole vector.
// reset_wscale folds w into aw with BLAS daxpy; the x86-64 BLAS kernels fuse that multiply-add, so the fold is the one
// fused operation of the file (__fma_rn).  Everything else is rounded step by step, as the Cython is.
// w, aw and q stay in shared memory for the epoch when they fit (8 d bytes each), in global memory otherwise.
#include "bkm_common.cuh"

#include <cstring>

namespace bkm {
namespace {

constexpr int kThreads = 256;
constexpr int kTile = 1024;                       // row entries staged per pass of the dot chain
// staged per entry: x_j, w[idx] * x_j, x_j * x_j (float64) and idx (int32)
constexpr size_t kStageBytes = (size_t)kTile * (3 * sizeof(double) + sizeof(int));
constexpr size_t kSmemLimit = 220 * 1024;         // dynamic shared memory asked for at most (H100: 227 KB per CTA)
constexpr double kMaxDloss = 1e12;
constexpr double kResetWscale = 1e-9;

enum { L1 = 1, L2 = 2, ELASTICNET = 3 };
enum { CONSTANT = 1, OPTIMAL = 2, INVSCALING = 3, ADAPTIVE = 4, PA1 = 5, PA2 = 6 };

struct SgdArgs {
  const void* vals;            // dense X, or the CSR values
  const long long* crow;       // CSR only
  const long long* col;        // CSR only
  long long ldx;               // dense only
  long long n;
  int d;
  const int* order;
  const double* y;
  const double* sw;
  const double* eta;
  const double* cw;
  double* w;
  double* aw;
  double* q;
  double* st;
  int smem_vecs;               // 0: the vectors stay in global memory
  bkm_sgd_params prm;
};

// cy_gradient(y, p) of the losses of SGDClassifier / SGDRegressor (sklearn 1.9)
__device__ double sgd_dloss(int loss, double eps, double y, double p) {
  switch (loss) {
    case BKM_SGD_HINGE: {
      const double z = p * y;
      return z <= eps ? -y : 0.0;
    }
    case BKM_SGD_LOG: {                               // cgradient_half_binomial, y in {0, 1}
      if (p > -37) {
        const double e = exp(-p);
        return ((1 - y) - y * e) / (1 + e);
      }
      return exp(p) - y;
    }
    case BKM_SGD_MODIFIED_HUBER: {
      const double z = p * y;
      if (z >= 1.0) return 0.0;
      if (z >= -1.0) return 2.0 * (1.0 - z) * -y;
      return -4.0 * y;
    }
    case BKM_SGD_SQUARED_HINGE: {
      const double z = eps - p * y;
      return z > 0 ? -2 * y * z : 0.0;
    }
    case BKM_SGD_SQUARED_ERROR:
      return p - y;
    case BKM_SGD_HUBER: {
      const double r = p - y;
      if (fabs(r) <= eps) return r;
      return r >= 0 ? eps : -eps;
    }
    case BKM_SGD_EPS_INSENSITIVE:
      if (y - p > eps) return -1;
      if (p - y > eps) return 1;
      return 0;
    default: {                                        // BKM_SGD_SQ_EPS_INSENSITIVE
      const double z = y - p;
      if (z > eps) return -2 * (z - eps);
      if (z < -eps) return 2 * (-z - eps);
      return 0;
    }
  }
}

// cy_loss(y, p) of the losses the passive-aggressive rates use (hinge, epsilon_insensitive) and their squared forms
__device__ double sgd_loss(int loss, double eps, double y, double p) {
  switch (loss) {
    case BKM_SGD_HINGE: {
      const double z = p * y;
      return z <= eps ? eps - z : 0.0;
    }
    case BKM_SGD_SQUARED_HINGE: {
      const double z = eps - p * y;
      return z > 0 ? z * z : 0.0;
    }
    case BKM_SGD_EPS_INSENSITIVE: {
      const double r = fabs(y - p) - eps;
      return r > 0 ? r : 0;
    }
    case BKM_SGD_SQ_EPS_INSENSITIVE: {
      const double r = fabs(y - p) - eps;
      return r > 0 ? r * r : 0;
    }
    default:
      return 0.0;
  }
}

template <typename T, bool CSR>
__global__ void __launch_bounds__(kThreads) sgd_kernel(const SgdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* xv = reinterpret_cast<double*>(smem_raw);
  double* xp = xv + kTile;
  double* xs = xp + kTile;
  int* xi = reinterpret_cast<int*>(xs + kTile);
  double* vecs = reinterpret_cast<double*>(xi + kTile);
  __shared__ double sh[8];
  __shared__ int shi[4];
  __shared__ int nonfinite;

  const bkm_sgd_params& P = a.prm;
  const int p = blockIdx.x, tid = threadIdx.x, d = a.d;
  const long long n = a.n;
  const bool l1 = P.penalty == L1 || P.penalty == ELASTICNET;
  const bool avg = a.aw != nullptr;
  const bool pa = P.learning_rate >= PA1;
  const T* vals = reinterpret_cast<const T*>(a.vals);

  double* w = a.w + (size_t)p * d;
  double* aw = avg ? a.aw + (size_t)p * d : nullptr;
  double* q = l1 ? a.q + (size_t)p * d : nullptr;
  double* gw = w;
  double* gaw = aw;
  if (a.smem_vecs) {
    double* v = vecs;
    w = v;
    v += d;
    if (avg) {
      aw = v;
      v += d;
    }
    if (l1) q = v;
    for (int j = tid; j < d; j += kThreads) {
      w[j] = gw[j];
      if (avg) aw[j] = gaw[j];
    }
  }
  if (l1)
    for (int j = tid; j < d; j += kThreads) q[j] = 0.0;
  if (tid == 0) nonfinite = 0;
  __syncthreads();

  // the scalar state of _plain_sgd and WeightVector, kept by thread 0
  double wscale = 1.0, intercept = a.st[4 * p], avg_intercept = a.st[4 * p + 1];
  double average_a = 0.0, average_b = 1.0, u = 0.0, t = P.t0, eta = P.eta0;
  const double l1_ratio = P.penalty == L2 ? 0.0 : (P.penalty == L1 ? 1.0 : P.l1_ratio);
  const double weight_pos = a.cw[2 * p], weight_neg = a.cw[2 * p + 1];
  const int* order = a.order + (size_t)p * n;
  const double* yp = a.y + (size_t)p * n;

  for (long long i = 0; i < n; ++i) {
    const long long r = order[i];
    long long beg, nnz;
    if (CSR) {
      beg = a.crow[r];
      nnz = a.crow[r + 1] - beg;
    } else {
      beg = r * a.ldx;
      nnz = d;
    }
    // 1. the dot product (and the squared norm of PA): one chain each, in stored order
    double acc = 0.0, sq = 0.0;
    for (long long t0 = 0; t0 < nnz; t0 += kTile) {
      const int m = (int)(nnz - t0 < kTile ? nnz - t0 : kTile);
      for (int j = tid; j < m; j += kThreads) {
        const double x = (double)vals[beg + t0 + j];
        const int idx = CSR ? (int)a.col[beg + t0 + j] : (int)(t0 + j);
        xv[j] = x;
        xi[j] = idx;
        xp[j] = __dmul_rn(w[idx], x);
        if (pa) xs[j] = __dmul_rn(x, x);
      }
      __syncthreads();
      if (tid == 0) {
#pragma unroll 8
        for (int j = 0; j < m; ++j) {
          acc = __dadd_rn(acc, xp[j]);
          if (pa) sq = __dadd_rn(sq, xs[j]);
        }
      }
      if (t0 + kTile < nnz) __syncthreads();      // the next tile overwrites the staged entries
    }
    // 2. the scalar step
    if (tid == 0) {
      const double pred = acc * wscale + intercept;
      if (P.learning_rate == OPTIMAL)
        eta = 1.0 / (P.alpha * (P.optimal_init + t - 1));
      else if (P.learning_rate == INVSCALING)
        eta = a.eta[i];
      const double yv = yp[r];
      const double swv = a.sw ? a.sw[r] : 1.0;
      const double class_weight = yv > 0.0 ? weight_pos : weight_neg;
      double update = 0.0;
      int skip = 0;
      if (P.learning_rate == PA1) {
        update = sq;
        if (update == 0) {
          skip = 1;
        } else {
          const double v = sgd_loss(P.loss, P.epsilon, yv, pred) / update;
          update = v < P.eta0 ? v : P.eta0;
        }
      } else if (P.learning_rate == PA2) {
        update = sq;
        update = sgd_loss(P.loss, P.epsilon, yv, pred) / (update + 0.5 / P.eta0);
      } else {
        double dloss = sgd_dloss(P.loss, P.epsilon, yv, pred);
        if (dloss < -kMaxDloss)
          dloss = -kMaxDloss;
        else if (dloss > kMaxDloss)
          dloss = kMaxDloss;
        update = -eta * dloss;
      }
      int reset = 0;
      if (!skip) {
        if (pa) {
          if (P.loss == BKM_SGD_HINGE)
            update *= yv;
          else if (yv - pred < 0)
            update *= -1;
        }
        update *= class_weight * swv;
        if (P.penalty >= L2) {                    // w.scale(max(0, 1 - (1 - l1_ratio) eta alpha))
          const double v = 1.0 - ((1.0 - l1_ratio) * eta * P.alpha);
          wscale *= v > 0 ? v : 0;
          if (wscale < kResetWscale) {
            reset = 1;
            sh[2] = wscale;
            sh[3] = average_a;
            sh[4] = average_b;
            average_a = 0.0;
            average_b = 1.0;
            wscale = 1.0;
          }
        }
        sh[0] = update / wscale;                  // w.add: val * (c / wscale)
        sh[1] = average_a;                        // w.add_average: average_a * val * (-c / wscale)
        sh[7] = -update / wscale;
        if (P.fit_intercept == 1) {
          const double intercept_update = update;
          if (intercept_update != 0) intercept += intercept_update * P.intercept_decay;
        }
        int do_avg = 0;
        if (0 < P.average && P.average <= t) {
          do_avg = 1;
          const double num_iter = t - P.average + 1;
          const double mu = 1.0 / num_iter;
          if (num_iter > 1) average_b /= (1.0 - mu);
          average_a += mu * average_b * wscale;
          avg_intercept += ((intercept - avg_intercept) / (t - P.average + 1));
        }
        if (l1) u += (l1_ratio * eta * P.alpha);
        sh[5] = wscale;
        sh[6] = u;
        shi[2] = update != 0.0;
        shi[3] = do_avg;
        t += 1;
      }
      shi[0] = skip;
      shi[1] = reset;
    }
    __syncthreads();
    if (shi[0]) continue;                         // PA-I on an all-zero row: the row is skipped (t unchanged)
    if (shi[1]) {                                 // WeightVector.reset_wscale inside w.scale
      const double ws = sh[2], aa = sh[3], inv_b = 1.0 / sh[4];
      for (int j = tid; j < d; j += kThreads) {
        if (avg) aw[j] = __fma_rn(aa, w[j], aw[j]) * inv_b;   // BLAS daxpy (fused on FMA hosts), dscal
        w[j] = w[j] * ws;
      }
      __syncthreads();
    }
    // 3. the per-entry updates: w.add, w.add_average, l1penalty, in that order for each entry
    const double c_w = sh[0], avg_a = sh[1], c_a = sh[7], ws = sh[5], uu = sh[6];
    const bool do_add = shi[2], do_avg = shi[3];
    const bool staged = nnz <= kTile;
    for (long long j = tid; j < nnz; j += kThreads) {
      const double x = staged ? xv[j] : (double)vals[beg + j];
      const int idx = staged ? xi[j] : (CSR ? (int)a.col[beg + j] : (int)j);
      if (do_add) w[idx] += x * c_w;
      if (do_avg) aw[idx] += avg_a * x * c_a;
      if (l1) {
        const double z = w[idx];
        if (ws * z > 0.0) {
          const double v = w[idx] - ((uu + q[idx]) / ws);
          w[idx] = v > 0.0 ? v : 0.0;
        } else if (ws * z < 0.0) {
          const double v = w[idx] + ((uu - q[idx]) / ws);
          w[idx] = v < 0.0 ? v : 0.0;
        }
        q[idx] += ws * (w[idx] - z);
      }
    }
    __syncthreads();                              // before the next row's entries are staged
  }

  // end of the epoch: the non-finite test on the unscaled weights, then reset_wscale
  for (int j = tid; j < d; j += kThreads)
    if (!isfinite(w[j])) nonfinite = 1;
  if (tid == 0) {
    sh[2] = wscale;
    sh[3] = average_a;
    sh[4] = average_b;
    if (!isfinite(intercept)) nonfinite = 1;
  }
  __syncthreads();
  const bool bad = nonfinite != 0;
  if (!bad) {
    const double ws = sh[2], aa = sh[3], inv_b = 1.0 / sh[4];
    for (int j = tid; j < d; j += kThreads) {
      if (avg) aw[j] = __fma_rn(aa, w[j], aw[j]) * inv_b;   // BLAS daxpy (fused on FMA hosts), dscal
      w[j] = w[j] * ws;
    }
  }
  if (a.smem_vecs) {
    __syncthreads();
    for (int j = tid; j < d; j += kThreads) {
      gw[j] = w[j];
      if (avg) gaw[j] = aw[j];
    }
  }
  if (tid == 0) {
    a.st[4 * p] = intercept;
    a.st[4 * p + 1] = avg_intercept;
    a.st[4 * p + 2] = bad ? 1.0 : 0.0;
  }
}

int check_params(const bkm_sgd_params* prm, int64_t n, int d, int P, const int32_t* order, const double* y,
                 const double* eta, const double* cw, double* w, double* aw, double* q, double* st) {
  if (!prm || n < 0 || n > 0x7FFFFFFFLL || d <= 0 || P <= 0) return BKM_EINVAL;
  if ((int64_t)P * n > (1LL << 40)) return BKM_EINVAL;
  if (prm->loss < BKM_SGD_HINGE || prm->loss > BKM_SGD_SQ_EPS_INSENSITIVE) return BKM_EINVAL;
  if (prm->penalty < 0 || prm->penalty > ELASTICNET) return BKM_EINVAL;
  if (prm->learning_rate < CONSTANT || prm->learning_rate > PA2) return BKM_EINVAL;
  if (prm->learning_rate >= PA1 && prm->loss != BKM_SGD_HINGE && prm->loss != BKM_SGD_SQUARED_HINGE &&
      prm->loss != BKM_SGD_EPS_INSENSITIVE && prm->loss != BKM_SGD_SQ_EPS_INSENSITIVE)
    return BKM_EINVAL;
  if (!w || !st || !cw) return BKM_EINVAL;
  if ((prm->penalty == L1 || prm->penalty == ELASTICNET) && !q) return BKM_EINVAL;
  if (prm->average > 0 && !aw) return BKM_EINVAL;
  if (n > 0 && (!order || !y)) return BKM_EINVAL;
  if (n > 0 && prm->learning_rate == INVSCALING && !eta) return BKM_EINVAL;
  return 0;
}

template <typename T, bool CSR>
int launch(SgdArgs a, int P, cudaStream_t s) {
  const int nvec = 1 + (a.aw ? 1 : 0) + (a.q ? 1 : 0);
  const size_t vec_bytes = (size_t)nvec * a.d * sizeof(double);
  a.smem_vecs = kStageBytes + vec_bytes <= kSmemLimit ? nvec : 0;
  const size_t smem = kStageBytes + (a.smem_vecs ? vec_bytes : 0);
  BKM_CUDA_TRY(cudaFuncSetAttribute(sgd_kernel<T, CSR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sgd_kernel<T, CSR><<<P, kThreads, smem, s>>>(a);
  BKM_CUDA_TRY(cudaGetLastError());
  note_launch();
  return 0;
}

}  // namespace
}  // namespace bkm

using namespace bkm;

extern "C" int bkm_sgd_order(int64_t n, uint32_t seed, int32_t* out_host) {
  if (n < 0 || n > 0x7FFFFFFFLL || (n > 0 && !out_host)) return BKM_EINVAL;
  const int nn = (int)n;
  for (int i = 0; i < nn; ++i) out_host[i] = i;
  for (unsigned i = 0; (long long)i < (long long)nn - 1; ++i) {
    if (seed == 0) seed = 1;                       // our_rand_r, sklearn/utils/_random.pxd
    seed ^= (uint32_t)(seed << 13);
    seed ^= (uint32_t)(seed >> 17);
    seed ^= (uint32_t)(seed << 5);
    const uint32_t rnd = seed % (0x7FFFFFFFu + 1u);
    const unsigned j = i + rnd % ((unsigned)nn - i);
    const int32_t tmp = out_host[i];
    out_host[i] = out_host[j];
    out_host[j] = tmp;
  }
  return 0;
}

extern "C" int bkm_sgd_block(const void* X, int64_t n, int d, int64_t ldx, int x_dtype, const int32_t* order,
                             const double* y, const double* sample_weight, const double* eta, const double* cw, int P,
                             const bkm_sgd_params* params_host, double* w, double* aw, double* q, double* st,
                             void* stream) {
  int rc = check_params(params_host, n, d, P, order, y, eta, cw, w, aw, q, st);
  if (rc) return rc;
  if (x_dtype != BKM_F32 && x_dtype != BKM_F64) return BKM_EDTYPE;
  if (ldx < d || (n > 0 && !X)) return BKM_EINVAL;
  if (n == 0) return 0;
  SgdArgs a;
  std::memset(&a, 0, sizeof(a));
  a.vals = X;
  a.ldx = ldx;
  a.n = n;
  a.d = d;
  a.order = order;
  a.y = y;
  a.sw = sample_weight;
  a.eta = eta;
  a.cw = cw;
  a.w = w;
  a.aw = params_host->average > 0 ? aw : nullptr;
  a.q = (params_host->penalty == L1 || params_host->penalty == ELASTICNET) ? q : nullptr;
  a.st = st;
  a.prm = *params_host;
  cudaStream_t s = (cudaStream_t)stream;
  return x_dtype == BKM_F32 ? launch<float, false>(a, P, s) : launch<double, false>(a, P, s);
}

extern "C" int bkm_sgd_csr_block(const int64_t* crow, const int64_t* col, const void* val, int val_dtype, int64_t n,
                                 int d, int64_t nnz, const int32_t* order, const double* y,
                                 const double* sample_weight, const double* eta, const double* cw, int P,
                                 const bkm_sgd_params* params_host, double* w, double* aw, double* q, double* st,
                                 void* stream) {
  int rc = check_params(params_host, n, d, P, order, y, eta, cw, w, aw, q, st);
  if (rc) return rc;
  if (val_dtype != BKM_F32 && val_dtype != BKM_F64) return BKM_EDTYPE;
  if (nnz < 0 || (n > 0 && !crow) || (nnz > 0 && (!col || !val))) return BKM_EINVAL;
  if (n == 0) return 0;
  SgdArgs a;
  std::memset(&a, 0, sizeof(a));
  a.vals = val;
  a.crow = reinterpret_cast<const long long*>(crow);
  a.col = reinterpret_cast<const long long*>(col);
  a.n = n;
  a.d = d;
  a.order = order;
  a.y = y;
  a.sw = sample_weight;
  a.eta = eta;
  a.cw = cw;
  a.w = w;
  a.aw = params_host->average > 0 ? aw : nullptr;
  a.q = (params_host->penalty == L1 || params_host->penalty == ELASTICNET) ? q : nullptr;
  a.st = st;
  a.prm = *params_host;
  cudaStream_t s = (cudaStream_t)stream;
  return val_dtype == BKM_F32 ? launch<float, true>(a, P, s) : launch<double, true>(a, P, s);
}

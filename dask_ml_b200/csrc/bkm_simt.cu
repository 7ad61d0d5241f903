// bkm_simt.cu — generic fused E+M chunk kernel on CUDA cores (any d, any k, fp32 or fp64).
//
// One launch per row chunk performs, for every row x of the chunk:
//   E-step  argmin_j ||x-c_j||^2 via ||c||^2 - 2 x.c (+||x||^2), lowest index on ties
//           (reference: sklearn pairwise_distances_argmin_min called per chunk at
//            dask_ml/metrics/pairwise.py:35-38; clamp >= 0)
//   M-step  sums[label] += x, counts[label] += 1
//           (reference: _centers_dense dask_ml/cluster/k_means.py:572-582, da.bincount :548)
// Rows whose best/second-best margin is within the fp32 rounding bound are re-evaluated in
// float64 against the float64 centres so that labels agree with the reference's float64
// E-step except for genuine float64 near-ties.
//
// Data movement: a tile of TILE rows is staged once in shared memory with coalesced 16-byte
// loads; both the E-step and the M-step read it from there, so X is read from HBM exactly once
// per Lloyd iteration.  Centres, per-CTA sums and counts live in shared memory (SMEM mode) or,
// when k*d is too large for that, centres are read through L1 and sums go to float64 global
// atomics (GLOBAL mode: one slot adds the rows of the whole chunk, where an fp32 running sum of a
// dominant cluster would lose its low bits).
#include "bkm_common.cuh"
#include <math_constants.h>

namespace bkm {

static const int TILE = 256;   // rows per tile == threads per CTA
static const int NW = TILE / 32;

template <typename T> struct PsumT { typedef float type; };
template <> struct PsumT<double> { typedef double type; };

template <typename T> __device__ __forceinline__ void ld4(const T* p, T (&v)[4]);
template <> __device__ __forceinline__ void ld4<float>(const float* p, float (&v)[4]) {
  float4 t = *reinterpret_cast<const float4*>(p);
  v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
template <> __device__ __forceinline__ void ld4<double>(const double* p, double (&v)[4]) {
  double2 a = reinterpret_cast<const double2*>(p)[0];
  double2 b = reinterpret_cast<const double2*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
}
template <typename T> __device__ __forceinline__ T inf_of();
template <> __device__ __forceinline__ float inf_of<float>() { return CUDART_INF_F; }
template <> __device__ __forceinline__ double inf_of<double>() { return CUDART_INF; }

// Row pitch (in elements) of the staged X tile: 16-byte units per row must be odd so that
// "thread r reads 16 bytes of row r" is bank-conflict free.
template <typename T> __host__ __device__ inline int tile_pitch(int d4) {
  int units = d4 * (int)sizeof(T) / 16;
  units |= 1;
  return units * 16 / (int)sizeof(T);
}

struct SimtSmem {
  size_t off_cs, off_cns, off_xs, off_lab, off_red2, off_flist, off_sums, off_cnts, off_misc, total;
  int rt;     // rows per tile (<= TILE; smaller for very wide rows so that the staged tile still fits shared memory)
};
static const size_t kSmemBudget = 227 * 1024;

template <typename T>
static inline SimtSmem simt_smem(int k, int d, int J, bool mstep, bool global_mode, int rt = TILE) {
  typedef typename PsumT<T>::type PS;
  int d4 = (d + 3) / 4 * 4;
  int kJ = (k + J - 1) / J * J;
  int pitch = tile_pitch<T>(d4);
  SimtSmem S; size_t o = 0;
  S.off_cs = o;   if (!global_mode) o += (size_t)kJ * d4 * sizeof(T);
  o = align_up(o, 16);
  S.off_cns = o;  o += (size_t)kJ * sizeof(T); o = align_up(o, 16);
  S.rt = rt;
  S.off_xs = o;   o += (size_t)rt * pitch * sizeof(T); o = align_up(o, 16);
  S.off_lab = o;  o += TILE * 4;
  S.off_red2 = o; o += TILE * 8;
  S.off_flist = o; o += TILE * 4;
  S.off_sums = o; if (mstep && !global_mode) o += (size_t)k * d * sizeof(PS);
  o = align_up(o, 16);
  S.off_cnts = o; if (mstep) o += (size_t)k * 4;
  o = align_up(o, 16);
  S.off_misc = o; o += 256;
  S.total = o;
  return S;
}

// Centres + per-CTA sums resident in shared memory (SMEM mode) need room for at least a 32-row tile next to them;
// otherwise centres are read through L1/L2 and the sums go to global atomics (GLOBAL mode).
template <typename T>
static inline bool simt_mode_global(int k, int d, int J, bool mstep) {
  return simt_smem<T>(k, d, J, mstep, false, 32).total > kSmemBudget;
}

template <typename T, int J, bool MSTEP, bool GLOBAL, bool SMALLK>
__global__ void __launch_bounds__(TILE)
simt_chunk_kernel(ChunkArgs a, SimtSmem S) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  typedef typename PsumT<T>::type PS;
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d, k = a.k, d4 = a.L.d4;
  const int kJ = (k + J - 1) / J * J;
  const int pitch = tile_pitch<T>(d4);
  const int nch = d4 / 4;

  T* cs = reinterpret_cast<T*>(smem + S.off_cs);
  T* cns = reinterpret_cast<T*>(smem + S.off_cns);
  T* xs = reinterpret_cast<T*>(smem + S.off_xs);
  int* lab_s = reinterpret_cast<int*>(smem + S.off_lab);
  double* red2_s = reinterpret_cast<double*>(smem + S.off_red2);
  int* flist = reinterpret_cast<int*>(smem + S.off_flist);
  PS* sums_s = reinterpret_cast<PS*>(smem + S.off_sums);
  int* cnts_s = reinterpret_cast<int*>(smem + S.off_cnts);
  int* misc = reinterpret_cast<int*>(smem + S.off_misc);   // [0]=nflag, [8..]: reduce scratch

  const T* gC = reinterpret_cast<const T*>(a.pack + a.L.off_cT);      // [k][d4]
  const T* gCn = reinterpret_cast<const T*>(a.pack + a.L.off_cnT);    // [k]
  const double* gC64 = reinterpret_cast<const double*>(a.pack + a.L.off_c64);
  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const T* X = reinterpret_cast<const T*>(a.X);

  // ---- one-time staging of centres, ||c||^2, zeroing of accumulators and tile padding ----
  if (!GLOBAL) {
    for (int i = tid; i < kJ * d4; i += TILE) cs[i] = (i < k * d4) ? gC[i] : T(0);
  }
  for (int i = tid; i < kJ; i += TILE) cns[i] = (i < k) ? gCn[i] : inf_of<T>();
  if (MSTEP) {
    if (!GLOBAL) for (int i = tid; i < k * d; i += TILE) sums_s[i] = PS(0);
    for (int i = tid; i < k; i += TILE) cnts_s[i] = 0;
  }
  const int RT = S.rt;
  for (int i = tid; i < RT * pitch; i += TILE) xs[i] = T(0);
  const T cnmax = (T)hdr->cn_max;
  double inertia_acc = 0.0;
  // Few clusters (k <= 32, d <= 16; BASELINE C4 / C1): lane j of every warp owns cluster j and keeps the sums of the
  // rows of ITS warp's 32-row slice in registers — lanes work on different rows at the same time, where the general
  // M-step below walks the rows one by one.  Folded into the shared-memory sums once, at the end of the kernel.
  // (a separate instantiation, so that the general kernel does not carry the 16 accumulator registers)
  constexpr bool smallk = SMALLK;
  PS lacc[SMALLK ? 16 : 1];
#pragma unroll
  for (int i = 0; i < (SMALLK ? 16 : 1); ++i) lacc[i] = PS(0);
  int lcnt = 0;
  __syncthreads();

  const long long ntiles = (a.n + RT - 1) / RT;
  // rows with a small padding (the 16-byte pitch the tensor path wants, e.g. 13 -> 16) are streamed like
  // contiguous ones: the whole [rows][ldx] block is read with 16-byte loads and the padding is dropped
  const int L = (int)a.ldx;
  const bool flat_ok = ((reinterpret_cast<uintptr_t>(X) & 15) == 0) &&
                       (a.ldx == d || (a.ldx <= d + 8 && (a.ldx * sizeof(T)) % 16 == 0));

  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long r0 = tile * RT;
    const int rows = (int)min((long long)RT, a.n - r0);

    // ---- stage the tile: coalesced loads, [row][pitch] layout in smem ----
    if (flat_ok && ((r0 * (long long)L * (long long)sizeof(T)) & 15) == 0) {
      const int per16 = 16 / (int)sizeof(T);
      const long long nelem = (long long)rows * L;
      const T* src = X + r0 * (long long)L;     // 16-byte aligned (checked above)
      const long long nvec = nelem / per16;
      for (long long v = tid; v < nvec; v += TILE) {
        T e[4];
        if (sizeof(T) == 4) {
          float4 t = __ldcs(reinterpret_cast<const float4*>(src) + v);
          e[0] = (T)t.x; e[1] = (T)t.y; e[2] = (T)t.z; e[3] = (T)t.w;
        } else {
          double2 t = __ldcs(reinterpret_cast<const double2*>(src) + v);
          e[0] = (T)t.x; e[1] = (T)t.y;
        }
        long long e0 = v * per16;
        int row = (int)(e0 / L);
        int col = (int)(e0 - (long long)row * L);
#pragma unroll
        for (int q = 0; q < per16; ++q) {
          if (col < d) xs[row * pitch + col] = e[q];
          if (++col == L) { col = 0; ++row; }
        }
      }
      for (long long e0 = nvec * per16 + tid; e0 < nelem; e0 += TILE) {
        int row = (int)(e0 / L);
        int col = (int)(e0 - (long long)row * L);
        if (col < d) xs[row * pitch + col] = src[e0];
      }
    } else {
      for (int r = warp; r < rows; r += NW) {
        const T* src = X + (r0 + r) * a.ldx;
        for (int i = lane; i < d; i += 32) xs[r * pitch + i] = src[i];
      }
    }
    if (tid == 0) misc[0] = 0;
    __syncthreads();

    // ---- E-step: thread r owns row r ----
    const bool valid = tid < rows;
    T best = inf_of<T>(), second = inf_of<T>();
    int bj = 0;
    T xn = T(0), dexact = T(0);
    int my_slot = -1;
    if (valid) {
      const T* xr = xs + tid * pitch;
      for (int ch = 0; ch < nch; ++ch) {
        T xv[4]; ld4<T>(xr + ch * 4, xv);
        xn = fma(xv[0], xv[0], fma(xv[1], xv[1], fma(xv[2], xv[2], fma(xv[3], xv[3], xn))));
      }
      for (int jg = 0; jg < kJ; jg += J) {
        T acc[J];
#pragma unroll
        for (int j = 0; j < J; ++j) acc[j] = T(0);
        const T* cb = (GLOBAL ? gC : cs) + (size_t)jg * d4;
        for (int ch = 0; ch < nch; ++ch) {
          T xv[4]; ld4<T>(xr + ch * 4, xv);
#pragma unroll
          for (int j = 0; j < J; ++j) {
            T cv[4];
            if (GLOBAL) {
              if (jg + j < k) ld4<T>(cb + (size_t)j * d4 + ch * 4, cv);
              else { cv[0] = cv[1] = cv[2] = cv[3] = T(0); }
            } else {
              ld4<T>(cb + (size_t)j * d4 + ch * 4, cv);
            }
            acc[j] = fma(xv[0], cv[0], fma(xv[1], cv[1], fma(xv[2], cv[2], fma(xv[3], cv[3], acc[j]))));
          }
        }
#pragma unroll
        for (int j = 0; j < J; ++j) {
          T dist = fma(T(-2), acc[j], cns[jg + j]);
          if (dist < best) { second = best; best = dist; bj = jg + j; }
          else if (dist < second) { second = dist; }
        }
      }
      lab_s[tid] = bj;
      {
        // winning distance re-evaluated in direct form sum (x-c)^2: error relative to the distance
        // itself, not to ||x||^2 (no cancellation) -> rows that coincide with a centre give 0.
        const T* cw = (GLOBAL ? gC : cs) + (size_t)bj * d4;
        T s = T(0);
        for (int ch = 0; ch < nch; ++ch) {
          T xv[4], cv[4];
          ld4<T>(xr + ch * 4, xv);
          ld4<T>(cw + ch * 4, cv);
#pragma unroll
          for (int q = 0; q < 4; ++q) { T df = xv[q] - cv[q]; s = fma(df, df, s); }
        }
        dexact = s;
      }
      if (a.tau > 0.f && k > 1) {
        T bound = (T)a.tau * (xn + cnmax);
        // near-tie, NaN, or a row outside the fp32 magnitude window (a.tau > 0: fp32 rows only)
        if (!(second - best > bound) || !fp32_norm_in_window((float)(xn + cnmax))) {
          my_slot = atomicAdd(&misc[0], 1);
          flist[my_slot] = tid;
        }
      }
    } else {
      lab_s[tid] = -1;
    }
    __syncthreads();

    // ---- float64 re-check of near-tie rows, whole CTA cooperates on each flagged row ----
    const int nflag = misc[0];
    for (int f = 0; f < nflag; ++f) {
      const int r = flist[f];
      const T* xr = xs + r * pitch;
      double bd = CUDART_INF; int bjj = 0x7fffffff;
      for (int j = tid; j < k; j += TILE) {
        const double* c = gC64 + (size_t)j * d;
        double s = 0.0;
        for (int i = 0; i < d; ++i) { double df = (double)xr[i] - c[i]; s = fma(df, df, s); }
        if (s < bd) { bd = s; bjj = j; }
      }
      // block argmin, lexicographic (distance, index)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        double od = __shfl_xor_sync(0xffffffffu, bd, o);
        int oj = __shfl_xor_sync(0xffffffffu, bjj, o);
        if (od < bd || (od == bd && oj < bjj)) { bd = od; bjj = oj; }
      }
      double* wd = reinterpret_cast<double*>(misc + 8);
      int* wj = misc + 8 + 2 * NW;
      if (lane == 0) { wd[warp] = bd; wj[warp] = bjj; }
      __syncthreads();
      if (tid == 0) {
        double fd = wd[0]; int fj = wj[0];
        for (int w = 1; w < NW; ++w)
          if (wd[w] < fd || (wd[w] == fd && wj[w] < fj)) { fd = wd[w]; fj = wj[w]; }
        // a row with no finite distance (NaN or +-inf entries) kept no centre: label 0, as the streaming and bf16
        // kernels give it (the M-step indexes the sums by this label)
        lab_s[r] = fj == 0x7fffffff ? 0 : fj; red2_s[f] = fd;
      }
      __syncthreads();
    }

    // ---- outputs of the E-step ----
    if (valid) {
      double d2;
      int lbl = lab_s[tid];
      if (my_slot >= 0) d2 = red2_s[my_slot];
      else d2 = (double)dexact;
      double outv = a.squared ? d2 : sqrt(d2);
      inertia_acc += outv;
      if (a.labels) a.labels[r0 + tid] = lbl;
      if (a.min_out) reinterpret_cast<T*>(a.min_out)[r0 + tid] = (T)outv;
    }

    // ---- M-step: warp w owns clusters c with c % NW == w; no atomics in SMEM mode ----
    if (MSTEP && smallk) {
      const int rbase = warp * 32;
      const int ml = (rbase + lane < rows) ? lab_s[rbase + lane] : -1;
      unsigned mine = 0;                                   // rows of this warp's slice that belong to cluster `lane`
      for (int j = 0; j < k; ++j) {
        const unsigned mj = __ballot_sync(0xffffffffu, ml == j);
        if (lane == j) mine = mj;
      }
      while (mine) {
        const int b = __ffs(mine) - 1; mine &= mine - 1;
        const T* xr = xs + (rbase + b) * pitch;
#pragma unroll
        for (int i = 0; i < (SMALLK ? 16 : 1); ++i) if (i < d) lacc[i] += (PS)xr[i];
        ++lcnt;
      }
    } else if (MSTEP) {
      for (int base = 0; base < rows; base += 32) {
        int ml = (base + lane < rows) ? lab_s[base + lane] : -1;
        bool mine = GLOBAL ? (ml >= 0 && ((base >> 5) % NW) == warp) : (ml >= 0 && (ml % NW) == warp);
        unsigned m = __ballot_sync(0xffffffffu, mine);
        while (m) {
          int b = __ffs(m) - 1; m &= m - 1;
          int c = __shfl_sync(0xffffffffu, ml, b);
          const T* xr = xs + (base + b) * pitch;
          if (GLOBAL) {
            double* g = reinterpret_cast<double*>(a.psum) + (size_t)c * d;
            for (int i = lane; i < d; i += 32) atomicAdd(g + i, (double)xr[i]);
            if (lane == 0) atomicAdd(&cnts_s[c], 1);
          } else {
            PS* sr = sums_s + (size_t)c * d;
            for (int i = lane; i < d; i += 32) sr[i] += (PS)xr[i];
            if (lane == 0) cnts_s[c] += 1;
          }
        }
      }
    }
    __syncthreads();
  }

  // ---- flush per-CTA partials ----
  if (MSTEP && smallk) {
    // warps add their lane-resident sums in warp order (fixed order: reproducible)
    for (int w = 0; w < NW; ++w) {
      if (warp == w && lane < k) {
#pragma unroll
        for (int i = 0; i < (SMALLK ? 16 : 1); ++i) if (i < d) sums_s[lane * d + i] += lacc[i];
        cnts_s[lane] += lcnt;
      }
      __syncthreads();
    }
  }
  if (MSTEP) {
    if (!GLOBAL) {
      PS* g = reinterpret_cast<PS*>(a.psum) + (size_t)blockIdx.x * k * d;
      for (int i = tid; i < k * d; i += TILE) g[i] = sums_s[i];
    }
    int* gc = a.pcnt + (size_t)blockIdx.x * k;
    for (int i = tid; i < k; i += TILE) gc[i] = cnts_s[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) inertia_acc += __shfl_xor_sync(0xffffffffu, inertia_acc, o);
  double* wd = reinterpret_cast<double*>(misc + 8);
  if (lane == 0) wd[warp] = inertia_acc;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int w = 0; w < NW; ++w) s += wd[w];
    a.pin[blockIdx.x] = s;
  }
}

// Rows per tile: TILE unless the staged rows would not fit next to the other buffers (very wide rows: d in the hundreds
// or thousands run with fewer rows per tile; the idle threads of the thread-per-row E-step are the price).
template <typename T>
static int pick_rt(int k, int d, int J, bool mstep, bool global_mode) {
  int rt = TILE;
  while (rt > 1 && simt_smem<T>(k, d, J, mstep, global_mode, rt).total > kSmemBudget) rt = rt > 32 ? rt - 32 : rt / 2;
  return rt;
}

// The configuration of one call: centres per register block, SMEM or GLOBAL mode, the lane-owns-cluster M-step, and the
// shared-memory layout with its row tile.  The launch and bkm_debug_core_layout both take it from here.
struct SimtPlan {
  int J;
  bool global_mode, smallk;
  SimtSmem S;
};

template <typename T>
static SimtPlan simt_plan(int k, int d, bool mstep) {
  SimtPlan p;
  const int waste8 = (k + 7) / 8 * 8 - k, waste16 = (k + 15) / 16 * 16 - k;
  p.J = (waste16 <= waste8 && sizeof(T) == 4) ? 16 : 8;
  p.global_mode = simt_mode_global<T>(k, d, p.J, mstep);
  p.smallk = mstep && !p.global_mode && k <= 32 && d <= 16;
  p.S = simt_smem<T>(k, d, p.J, mstep, p.global_mode, pick_rt<T>(k, d, p.J, mstep, p.global_mode));
  return p;
}

template <typename T, int J, bool MSTEP, bool GLOBAL, bool SMALLK = false>
static int launch_one(const ChunkArgs& a, const SimtSmem& S, int sm_count, int* grid_out, cudaStream_t s) {
  if (S.total > kSmemBudget) return BKM_EUNSUPPORTED;
  auto kern = simt_chunk_kernel<T, J, MSTEP, GLOBAL, SMALLK>;
  BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S.total));
  int occ = 0;
  BKM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, TILE, S.total));
  if (occ < 1) return BKM_EUNSUPPORTED;
  long long ntiles = (a.n + S.rt - 1) / S.rt;
  long long grid = (long long)sm_count * occ;
  if (MSTEP && !GLOBAL && grid > a.psum_slots) grid = a.psum_slots;
  if (grid > a.part_slots) grid = a.part_slots;
  if (grid > ntiles) grid = ntiles;
  if (grid < 1) grid = 1;
  *grid_out = (int)grid;
  kern<<<(int)grid, TILE, S.total, s>>>(a, S);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// In GLOBAL mode the kernel accumulates into psum slot 0 with float64 atomics (fp32 inputs too): the
// caller zeroes it and reduce_partials reads it as a single float64 partial.  grid_out is returned
// negative in that case.
template <typename T>
static int launch_T(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  const SimtPlan p = simt_plan<T>(a.k, a.d, mstep);
  const SimtSmem& S = p.S;
  if (p.global_mode && mstep) {
    BKM_CUDA_TRY(cudaMemsetAsync(a.psum, 0, (size_t)a.k * a.d * sizeof(double), s));
    note_launch();
  }
  int rc;
#define BKM_DISPATCH(JJ)                                                                           \
  if (mstep) {                                                                                     \
    if (p.global_mode) rc = launch_one<T, JJ, true, true>(a, S, sm_count, grid_out, s);            \
    else if (p.smallk) rc = launch_one<T, JJ, true, false, true>(a, S, sm_count, grid_out, s);     \
    else rc = launch_one<T, JJ, true, false>(a, S, sm_count, grid_out, s);                         \
  } else {                                                                                         \
    if (p.global_mode) rc = launch_one<T, JJ, false, true>(a, S, sm_count, grid_out, s);           \
    else rc = launch_one<T, JJ, false, false>(a, S, sm_count, grid_out, s);                        \
  }
  if (p.J == 16) { BKM_DISPATCH(16) } else { BKM_DISPATCH(8) }
#undef BKM_DISPATCH
  if (rc == 0 && p.global_mode) *grid_out = -*grid_out;
  return rc;
}

int launch_simt(const ChunkArgs& a, bool mstep, int dtype, int sm_count, int* grid_out, cudaStream_t s) {
  return dtype == BKM_F32 ? launch_T<float>(a, mstep, sm_count, grid_out, s)
                          : launch_T<double>(a, mstep, sm_count, grid_out, s);
}

// bkm_debug_core_layout's generic-kernel fields: out[0] = 0, out[1..5] = {J, GLOBAL, SMALLK, rows per tile, staged tile
// pitch (elements)}, out[12] = dynamic shared-memory bytes
int simt_layout(int d, int k, int dtype, bool mstep, int* out13) {
  const bool f32 = dtype == BKM_F32;
  const SimtPlan p = f32 ? simt_plan<float>(k, d, mstep) : simt_plan<double>(k, d, mstep);
  if (p.S.total > kSmemBudget) return BKM_EUNSUPPORTED;
  const int d4 = (d + 3) / 4 * 4;
  out13[0] = 0;
  out13[1] = p.J;
  out13[2] = p.global_mode ? 1 : 0;
  out13[3] = p.smallk ? 1 : 0;
  out13[4] = p.S.rt;
  out13[5] = f32 ? tile_pitch<float>(d4) : tile_pitch<double>(d4);
  out13[12] = (int)p.S.total;
  return 0;
}

}  // namespace bkm

// bkm_tc.cu — fused E+M chunk kernel on the Hopper tensor cores (wgmma, sm_90a).
//
// Shapes: fp32 X with d <= 64 and a 16-byte aligned row pitch, k <= 256 (BASELINE config C2: 10M x 64, k = 256).
//
// Per 64-row tile of X a warpgroup computes  acc = (s X) . (-2 s C)^T  with the product as a split-fp16 triple
// (twice the TF32 rate):
//     Xhi.Bhi + Xhi.Blo + Xlo.Bhi        (hi = rn_fp16(v), lo = rn_fp16(v - hi): 22 significant bits)
// and adds s^2 ||c||^2 per column in fp32 in the epilogue.  s is a power of two chosen from the centres
// (PackHeader::scale) so that both operands sit in fp16's range; scaling by s is exact, so the result is the
// fp32-GEMM-class distance (~2^-22 relative error per product) and labels agree with the reference's float64 E-step
// (sklearn pairwise_distances_argmin_min, dask_ml/metrics/pairwise.py:35-38) except on near-ties, which are
// re-decided in float64 (as are rows whose scaled entries leave fp16's range).  The M-step (_centers_dense,
// dask_ml/cluster/k_means.py:572-582) is fused: rows are added into shared-memory per-CTA sums, X is read from HBM once.
//
// CTA = 2 warpgroups (1 CTA per SM).  Each warpgroup owns alternate 64-row tiles of the CTA and runs, per tile:
//   cp.async of the NEXT tile into its second stage (fp32 rows, zero-filled beyond n and d);
//   the fp16 (hi, lo) A fragments of s X built in registers (and ||s x||^2);
//   3 ceil(d/16) wgmma.m64nNk16 with B (= -2 s C as fp16 hi / lo, SWIZZLE_128B K-major) resident in shared memory;
//   the arg-min epilogue from the register accumulators (best, second best, near-tie test);
//   the winning distance in direct form (x - c)^2 in fp32, and the M-step.
// The M-step adds the tile's rows in row order into the CTA's sums; the two warpgroups take turns (named barriers),
// so every cluster's sum is formed in one fixed order and the sums are bit-reproducible.  One warpgroup's MMAs
// overlap the other's epilogue / M-step.
#include "bkm_common.cuh"
#include "bkm_wgmma.cuh"
#include <cuda_fp16.h>
#include <math_constants.h>

namespace bkm {

static const int TBM = 64;           // rows per warpgroup tile (wgmma M)
static const int XP = 72;            // fp32 row pitch of a staged X tile (16-byte multiple; rows 8 banks apart)
static const int TC_THREADS = 256;   // two warpgroups

struct TcCfg {
  int KS;        // MMA K-steps of 16 (ceil(d/16))
  int NP;        // padded centre count (multiple of 16, <= 256)
  uint32_t off_bhi, off_blo, off_x, off_sum, off_cn, off_cnt, off_lab, off_dp, off_red, total;
};

// The deferred-row re-check reports a failed fused kernel through this word (see tc_recheck_kernel); the wgmma kernel
// has no waits that can time out, so it stays 0 unless a debugging build sets it.
__device__ unsigned int g_tc_abort = 0;
__device__ unsigned int g_tc_dbg[64];

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);          // low half = lower column
  return *reinterpret_cast<const uint32_t*>(&h);
}

// XFORM: the epilogue writes the whole (rows x k) block of distances / kernel values instead of the arg-min
// (euclidean_distances, dask_ml/metrics/pairwise.py:69-97; rbf_kernel :131-139) — same MMAs, no M-step.
template <int N, bool MSTEP, bool WANT_DIST, bool XFORM>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_chunk_kernel(ChunkArgs a, TcCfg cfg) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  extern __shared__ __align__(1024) unsigned char smem[];
  constexpr bool HAS_M = MSTEP || WANT_DIST;
  const int tid = threadIdx.x, lane = tid & 31, wgi = tid >> 7, t = tid & 127, wq = t >> 5;
  const uint32_t sbase = smem_u32(smem);
  if (tid == 0 && (sbase & 1023)) __trap();                 // the swizzle pattern assumes 1024-byte aligned tiles
  const int KS = cfg.KS, d = a.d, k = a.k;
  float* cn_s = reinterpret_cast<float*>(smem + cfg.off_cn);          // [N] s^2 ||c||^2 (padded columns: 3e38)
  int* cnt_s = reinterpret_cast<int*>(smem + cfg.off_cnt);            // [N]
  float* sum_s = reinterpret_cast<float*>(smem + cfg.off_sum);        // [N][64]
  int* lab_s = reinterpret_cast<int*>(smem + cfg.off_lab) + wgi * TBM;        // label of each row of the tile, -1: none
  float* dp_s = reinterpret_cast<float*>(smem + cfg.off_dp) + wgi * 2 * TBM;  // [2][TBM] halves of the direct distances
  double* red_s = reinterpret_cast<double*>(smem + cfg.off_red);
  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const float sc = hdr->scale;

  // ---------------- setup: B tiles, column offsets, sums ----------------
  {
    // pack rows are 64 halves = 8 chunks of 16 bytes: chunk q of row r goes to its SWIZZLE_128B position
    const uint4* ghi = reinterpret_cast<const uint4*>(a.pack + a.L.off_bhi);
    const uint4* glo = reinterpret_cast<const uint4*>(a.pack + a.L.off_blo);
    for (int i = tid; i < N * 8; i += TC_THREADS) {
      const int r = i >> 3, q = i & 7;
      uint4 h = make_uint4(0u, 0u, 0u, 0u), l = h;
      if (r < a.L.kp) { h = ghi[i]; l = glo[i]; }
      *reinterpret_cast<uint4*>(smem + cfg.off_bhi + wg::sw128_chunk(r, q)) = h;
      *reinterpret_cast<uint4*>(smem + cfg.off_blo + wg::sw128_chunk(r, q)) = l;
    }
    // s^2 ||c_j||^2 from the pack's exact 3-way split [hi, mid, lo] (hi + mid + lo == the fp32 value)
    const float* bcn = reinterpret_cast<const float*>(a.pack + a.L.off_bcn);
    for (int j = tid; j < N; j += TC_THREADS) {
      float v = 3.0e38f;
      if (j < a.L.kp) { const float* p = bcn + (j >> 3) * 64 + (j & 7) * 4; v = (p[0] + p[1]) + p[2]; }
      cn_s[j] = v;
      cnt_s[j] = 0;
    }
    if (MSTEP)
      for (int i = tid; i < N * 64; i += TC_THREADS) sum_s[i] = 0.f;
    wg::fence_proxy_async();                                 // generic-proxy stores -> visible to wgmma
  }
  __syncthreads();

  const long long ntiles = (a.n + TBM - 1) / TBM;
  const long long my_tiles = blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const long long npairs = (my_tiles + 1) / 2;               // warpgroup w takes the CTA's tiles 2p + w
  const float* X = reinterpret_cast<const float*>(a.X);
  const uint32_t stage_bytes = TBM * XP * 4;
  const uint32_t xs_u32 = sbase + cfg.off_x + (uint32_t)wgi * 2u * stage_bytes;
  const float* xs_f = reinterpret_cast<const float*>(smem + cfg.off_x) + wgi * 2 * TBM * XP;
  const int nq = KS * 4;                                     // 16-byte chunks per staged row
  auto load_tile = [&](long long p, int stage) {
    const long long lt = 2 * p + wgi;
    if (lt < my_tiles) {
      const long long row0 = (blockIdx.x + lt * gridDim.x) * TBM;
      for (int i = t; i < TBM * nq; i += 128) {
        const int r = i / nq, col = (i - r * nq) * 4;
        const long long row = row0 + r;
        const int bytes = (row < a.n && col < d) ? min(16, (d - col) * 4) : 0;
        wg::cp16(xs_u32 + (uint32_t)stage * stage_bytes + (uint32_t)(r * XP + col) * 4u, bytes ? X + row * a.ldx + col : X, bytes);
      }
    }
    wg::cp_commit();
  };

  const int g = lane >> 2, c2 = (lane & 3) * 2;
  const int rA = wq * 16 + g;                                // this thread's accumulator rows: rA, rA + 8
  const uint64_t dbh = wg::desc_sw128(sbase + cfg.off_bhi), dbl = wg::desc_sw128(sbase + cfg.off_blo);
  const float cnmax = (float)(hdr->cn_max * (double)sc * (double)sc);
  double dsum = 0.0;

  load_tile(0, 0);
#pragma unroll 1
  for (long long p = 0; p < npairs; ++p) {
    const int stage = (int)(p & 1);
    load_tile(p + 1, stage ^ 1);
    wg::cp_wait1();
    wg::wg_sync(1 + wgi);                                    // tile p is in shared memory (every thread's copies)
    const long long lt = 2 * p + wgi;
    const bool has = lt < my_tiles;
    const long long row0 = (blockIdx.x + lt * gridDim.x) * TBM;
    const float* xs = xs_f + stage * TBM * XP;
    if (has) {
      // ---- s X -> fp16 (hi, lo) A fragments, ||s x||^2 of rows rA / rA + 8 ----
      uint32_t ahi[4][4], alo[4][4];
      float xn0 = 0.f, xn1 = 0.f;
#pragma unroll
      for (int s = 0; s < 4; ++s) {
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          ahi[s][h] = 0u; alo[s][h] = 0u;
          if (s < KS) {
            const float2 v = *reinterpret_cast<const float2*>(xs + (rA + (h & 1) * 8) * XP + s * 16 + c2 + (h >> 1) * 8);
            const float e0 = v.x * sc, e1 = v.y * sc;
            const __half2 hh = __floats2half2_rn(e0, e1);
            const float2 hf = __half22float2(hh);
            ahi[s][h] = *reinterpret_cast<const uint32_t*>(&hh);
            alo[s][h] = pack_half2(e0 - hf.x, e1 - hf.y);      // the subtraction is exact
            if (h & 1) xn1 = fmaf(e1, e1, fmaf(e0, e0, xn1));
            else xn0 = fmaf(e1, e1, fmaf(e0, e0, xn0));
          }
        }
      }
      xn0 += __shfl_xor_sync(0xffffffffu, xn0, 1); xn0 += __shfl_xor_sync(0xffffffffu, xn0, 2);
      xn1 += __shfl_xor_sync(0xffffffffu, xn1, 1); xn1 += __shfl_xor_sync(0xffffffffu, xn1, 2);

      // ---- acc = Xhi.Bhi + Xhi.Blo + Xlo.Bhi ----
      float acc[N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
      wg::fence();
#pragma unroll
      for (int s = 0; s < 4; ++s)
        if (s < KS) wg::Mma<N>::rs_f16(acc, ahi[s], dbh + (uint64_t)(2 * s), s > 0);
#pragma unroll
      for (int s = 0; s < 4; ++s)
        if (s < KS) wg::Mma<N>::rs_f16(acc, ahi[s], dbl + (uint64_t)(2 * s), 1);
#pragma unroll
      for (int s = 0; s < 4; ++s)
        if (s < KS) wg::Mma<N>::rs_f16(acc, alo[s], dbh + (uint64_t)(2 * s), 1);
      wg::commit();
      wg::wait_all();
      wg::pin(acc);

      if (XFORM) {
        // d^2 = (acc + s^2 ||c||^2 + ||s x||^2) / s^2, clamped at 0; mode 0: sqrt, 1: squared, 2: exp(-gamma d^2)
        const float inv_s2 = 1.0f / (sc * sc);
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(a.xf_out) & 7) == 0) && ((a.xf_ld & 1) == 0);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long row = row0 + rA + 8 * h;
          if (row >= a.n) continue;
          const float xn = h ? xn1 : xn0;
          float* orow = a.xf_out + row * a.xf_ld;
#pragma unroll
          for (int i = 0; i < N / 8; ++i) {
            const int col = 8 * i + c2;
            float o[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float d2 = fmaxf(((acc[4 * i + 2 * h + e] + cn_s[col + e]) + xn) * inv_s2, 0.f);
              o[e] = a.xf_mode == 0 ? sqrtf(d2) : (a.xf_mode == 1 ? d2 : __expf(-a.xf_gamma * d2));
            }
            if (vec_ok && col + 1 < k) __stcs(reinterpret_cast<float2*>(orow + col), make_float2(o[0], o[1]));
            else {
              if (col < k) orow[col] = o[0];
              if (col + 1 < k) orow[col + 1] = o[1];
            }
          }
        }
      } else {
        // ---- arg-min, near-tie test (bound = tau (||s x||^2 + max ||s c||^2)) ----
        wg::Best2 b0, b1;
        wg::tile_best2<N>(acc, cn_s, lane, b0, b1);
        if ((lane & 3) == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const wg::Best2 b = h ? b1 : b0;
            const float xn = h ? xn1 : xn0;
            const int r = rA + 8 * h;
            const long long row = row0 + r;
            // an entry beyond fp16's range (|s x| >= 65504 => xn >= 4.29e9) or a non-finite one: float64 path
            const bool out_of_range = !(xn < 4.29e9f);
            const bool tie = !(b.m2 > b.m1 + a.tau * (xn + cnmax)) || out_of_range;
            const bool valid = row < a.n;
            const bool flagged = valid && tie && k > 1;
            const int bj = (tie || b.j >= k) ? 0 : b.j;
            if (valid && !flagged && a.labels) a.labels[row] = bj;
            if (flagged) {
              // deferred: tc_recheck_kernel decides this row in float64 and adds its M-step contribution
              const int slot = atomicAdd(a.defer_cnt, 1);
              a.defer_idx[slot] = (int)row;
            }
            if (HAS_M) lab_s[r] = (valid && !flagged) ? bj : -1;
            if (MSTEP && valid && !flagged) atomicAdd(&cnt_s[bj], 1);
          }
        }
      }
    }
    if (HAS_M) {
      wg::wg_sync(1 + wgi);                                  // lab_s of the tile is complete
      if (WANT_DIST && has) {
        // winning distance in direct form sum (x - c)^2 (fp32 centres of the pack): thread (row r, feature half hh),
        // features visited in a per-row rotated order so that the 32 rows of a warp hit 32 different banks
        const int r = t & 63, hh = t >> 6;
        const int lab = lab_s[r];
        float s0 = 0.f, s1 = 0.f;
        if (lab >= 0) {
          const float* cr = reinterpret_cast<const float*>(a.pack + a.L.off_cT) + (size_t)lab * a.L.d4;
#pragma unroll 8
          for (int i = 0; i < 32; i += 2) {
            const int f0 = hh * 32 + ((i + r) & 31), f1 = hh * 32 + ((i + 1 + r) & 31);
            if (f0 < d) { const float e = xs[r * XP + f0] - cr[f0]; s0 = fmaf(e, e, s0); }
            if (f1 < d) { const float e = xs[r * XP + f1] - cr[f1]; s1 = fmaf(e, e, s1); }
          }
        }
        dp_s[hh * TBM + r] = s0 + s1;
        wg::wg_sync(1 + wgi);
        if (t < TBM && lab >= 0) {
          const float d2 = dp_s[t] + dp_s[TBM + t];
          const float outv = a.squared ? d2 : sqrtf(d2);
          dsum += (double)outv;
          if (a.min_out) reinterpret_cast<float*>(a.min_out)[row0 + t] = outv;
        }
      }
      if (MSTEP) {
        // turn order of the CTA's M-steps: warpgroup 0 tile p, warpgroup 1 tile p, warpgroup 0 tile p + 1, ...
        if (wgi == 1) bar_sync(3, 256);
        else if (p > 0) bar_sync(4, 256);
        if (has) {
          // thread (feature f, half h): half 0 adds rows 0-31, then half 1 rows 32-63, 8 rows at a time; when the 8
          // labels are distinct their read-modify-writes are independent, otherwise they run one after the other
          const int f = t & 63, h = t >> 6;
#pragma unroll 1
          for (int ph = 0; ph < 2; ++ph) {
            if (h == ph) {
#pragma unroll 1
              for (int r0 = 32 * ph; r0 < 32 * ph + 32; r0 += 8) {
                const int lr = lane < 8 ? lab_s[r0 + lane] : -2 - lane;
                const unsigned peers = __match_any_sync(0xffffffffu, lr);
                const bool conflict = __any_sync(0xffffffffu, lr >= 0 && __popc(peers) > 1);
                int l[8];
#pragma unroll
                for (int q = 0; q < 8; ++q) l[q] = __shfl_sync(0xffffffffu, lr, q);
                if (f < d) {
                  if (!conflict) {
                    float v[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) v[q] = l[q] >= 0 ? sum_s[l[q] * 64 + f] : 0.f;
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                      if (l[q] >= 0) sum_s[l[q] * 64 + f] = v[q] + xs[(r0 + q) * XP + f];
                  } else {
#pragma unroll
                    for (int q = 0; q < 8; ++q)
                      if (l[q] >= 0) sum_s[l[q] * 64 + f] += xs[(r0 + q) * XP + f];
                  }
                }
              }
            }
            if (ph == 0) wg::wg_sync(1 + wgi);
          }
        }
        __threadfence_block();
        if (wgi == 0) bar_arrive(3, 256);
        else if (p + 1 < npairs) bar_arrive(4, 256);
      }
    }
    wg::wg_sync(1 + wgi);                                    // the stage and lab_s may be refilled
  }

  // ---------------- teardown: per-CTA partials ----------------
  __syncthreads();
  if (MSTEP) {
    float* gs = reinterpret_cast<float*>(a.psum) + (size_t)blockIdx.x * k * d;
    for (int i = tid; i < k * d; i += TC_THREADS) {
      const int c = i / d;
      gs[i] = sum_s[c * 64 + (i - c * d)];
    }
    for (int c = tid; c < k; c += TC_THREADS) a.pcnt[(size_t)blockIdx.x * k + c] = cnt_s[c];
  }
  red_s[tid] = dsum;
  __syncthreads();
  if (tid == 0) {
    double tt = 0.0;
    for (int i = 0; i < TC_THREADS; ++i) tt += red_s[i];
    if (a.pin) a.pin[blockIdx.x] = tt;             // (the transform variant has no per-CTA partials)
  }
}

// ------------------------------------------------------------------------------------------
// Deferred float64 re-check.  Rows whose best/second margin was inside the rounding bound of the split-fp16
// product (or whose scaled entries left fp16's range) were left out of the fused kernel's outputs and M-step;
// here they are decided exactly: d2_j = sum_i (x_i - c_ji)^2 in float64 against the float64 centres
// (transposed, so that thread j <-> centre j reads are coalesced / conflict-free), lowest index on exact ties.  Their labels,
// distances and M-step contributions are then added (float64 atomics: order-insensitive to ~1e-16).
// ------------------------------------------------------------------------------------------
static const int RCK_ROWS = 8;      // deferred rows decided together by one CTA (the centres are read once per group)

__global__ void __launch_bounds__(256)
tc_recheck_kernel(ChunkArgs a, bool mstep, double* sums, unsigned long long* counts, double* dist_sum) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  __shared__ float xs[RCK_ROWS][64];
  __shared__ double wd[RCK_ROWS][8];
  __shared__ int wj[RCK_ROWS][8];
  __shared__ long long rows_s[RCK_ROWS];
  if (blockIdx.x == 0 && threadIdx.x == 0 && *(volatile unsigned int*)&g_tc_abort) {
    // a pipeline wait of the fused kernel timed out (see mbar_wait): its outputs are garbage.  Make that loud:
    // NaN sums / cost and a negative label instead of plausible numbers (bkm_debug_abort_code tells which wait).
    if (mstep && sums) sums[0] = CUDART_NAN;
    if (dist_sum) *dist_sum = CUDART_NAN;
    if (a.labels && a.n > 0) a.labels[0] = -1;
  }
  const int cnt = *a.defer_cnt;
  if ((int)blockIdx.x * RCK_ROWS >= cnt) return;
  const int k = a.k, d = a.d, tid = threadIdx.x, kp = a.L.kp, lane = tid & 31, wid = tid >> 5;
  // float64 centres, transposed [d][kp] by the pack: thread j <-> centre j reads are coalesced and hit L2
  // (every CTA reads the same 128 KB).
  const double* gT = reinterpret_cast<const double*>(a.pack + a.L.off_c64T);
  const float* X = reinterpret_cast<const float*>(a.X);
  for (int f0 = blockIdx.x * RCK_ROWS; f0 < cnt; f0 += gridDim.x * RCK_ROWS) {
    const int nr = min(RCK_ROWS, cnt - f0);
    __syncthreads();
    if (tid < RCK_ROWS) rows_s[tid] = tid < nr ? (long long)a.defer_idx[f0 + tid] : -1;
    __syncthreads();
    for (int e = tid; e < RCK_ROWS * 64; e += 256) {
      const int r = e >> 6, i = e & 63;
      xs[r][i] = (r < nr && i < d) ? X[rows_s[r] * a.ldx + i] : 0.f;
    }
    __syncthreads();
    // thread j: squared distances of the group's rows to centre j (two interleaved partial sums per row: the
    // order of the float64 additions is fixed, sum of even features + sum of odd features)
    double s0[RCK_ROWS], s1[RCK_ROWS];
#pragma unroll
    for (int r = 0; r < RCK_ROWS; ++r) { s0[r] = 0.0; s1[r] = 0.0; }
    const int j = tid;
    if (j < k) {
      int i = 0;
      for (; i + 1 < d; i += 2) {
        const double c0 = gT[(size_t)i * kp + j], c1 = gT[(size_t)(i + 1) * kp + j];
#pragma unroll
        for (int r = 0; r < RCK_ROWS; ++r) {
          const double d0 = (double)xs[r][i] - c0, d1 = (double)xs[r][i + 1] - c1;
          s0[r] = fma(d0, d0, s0[r]); s1[r] = fma(d1, d1, s1[r]);
        }
      }
      if (i < d) {
        const double c0 = gT[(size_t)i * kp + j];
#pragma unroll
        for (int r = 0; r < RCK_ROWS; ++r) { const double d0 = (double)xs[r][i] - c0; s0[r] = fma(d0, d0, s0[r]); }
      }
    }
#pragma unroll
    for (int r = 0; r < RCK_ROWS; ++r) {
      double bd = j < k ? s0[r] + s1[r] : CUDART_INF;
      int bj = j < k ? j : 0x7fffffff;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, bd, o);
        const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
        if (od < bd || (od == bd && oj < bj)) { bd = od; bj = oj; }
      }
      if (lane == 0) { wd[r][wid] = bd; wj[r][wid] = bj; }
    }
    __syncthreads();
    if (tid < nr) {
      const int r = tid;
      double fd = wd[r][0]; int fj = wj[r][0];
      for (int w = 1; w < 8; ++w) if (wd[r][w] < fd || (wd[r][w] == fd && wj[r][w] < fj)) { fd = wd[r][w]; fj = wj[r][w]; }
      const long long row = rows_s[r];
      const double outv = a.squared ? fd : sqrt(fd);
      if (a.labels) a.labels[row] = fj;
      if (a.min_out) reinterpret_cast<float*>(a.min_out)[row] = (float)outv;
      if (dist_sum) atomicAdd(dist_sum, outv);
      if (mstep) {
        if (a.counts_f64) atomicAdd(reinterpret_cast<double*>(counts) + fj, 1.0);
        else atomicAdd(counts + fj, 1ull);
      }
      wj[r][0] = fj;
    }
    __syncthreads();
    if (mstep)
      for (int e = tid; e < nr * 64; e += 256) {
        const int r = e >> 6, i = e & 63;
        if (i < d) atomicAdd(sums + (size_t)wj[r][0] * d + i, (double)xs[r][i]);
      }
  }
}

// Runs AFTER reduce_partials (which may overwrite the accumulators for the first chunk of an iteration): the deferred
// rows' contributions are added on top.
int launch_tc_recheck(const ChunkArgs& a, bool mstep, int sm_count, cudaStream_t s) {
  if (a.k <= 1) return 0;
  tc_recheck_kernel<<<sm_count * 4, 256, 0, s>>>(a, mstep, a.out_sums, (unsigned long long*)a.out_counts, a.out_dist_sum);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------ host
unsigned int tc_abort_code() {
  unsigned int v = 0;
  cudaMemcpyFromSymbol(&v, g_tc_abort, sizeof(v));
  return v;
}
int tc_trace(long long* out, int n) {
  (void)out; (void)n;
  return 0;
}
void tc_abort_detail(unsigned int* out64) { cudaMemcpyFromSymbol(out64, g_tc_dbg, 64 * sizeof(unsigned int)); }
// Clear the sticky abort word (after the host has reported it): later launches run normally again.
void tc_abort_reset() {
  const unsigned int z = 0;
  unsigned int zz[64] = {0};
  cudaMemcpyToSymbol(g_tc_abort, &z, sizeof(z));
  cudaMemcpyToSymbol(g_tc_dbg, zz, sizeof(zz));
}

bool tc_supported(int d, int k, int dtype) {
  // any d <= 64: columns beyond d are zero-filled when a tile is staged; what the staging copies do need is a
  // 16-byte row pitch and base (launch_tc returns BKM_EALIGN otherwise and the caller falls back to the CUDA-core
  // kernel), which the host side provides by uploading row chunks with a padded pitch (engine.CudaBackend.to_device)
  return dtype == BKM_F32 && d >= 1 && d <= 64 && k >= 1 && k <= 256;
}

static bool make_cfg(int d, int k, bool mstep, TcCfg* c) {
  c->KS = (d + 15) / 16;
  c->NP = (k + 15) / 16 * 16;
  const uint32_t N = (uint32_t)wg::mma_n(c->NP);
  uint32_t o = 0;
  c->off_bhi = o; o += N * 128u;                    // fp16 B tiles: N rows x 64 halves (one 128-byte swizzle atom)
  c->off_blo = o; o += N * 128u;
  c->off_x = o; o += 2u * 2u * TBM * XP * 4u;       // 2 warpgroups x 2 stages of fp32 X tiles
  c->off_sum = o; if (mstep) o += N * 64u * 4u;     // per-CTA sums [N][64]
  c->off_cn = o; o += N * 4u;
  c->off_cnt = o; o += N * 4u;
  c->off_lab = o; o += 2u * TBM * 4u;
  c->off_dp = o; o += 2u * 2u * TBM * 4u;
  c->off_red = o; o += TC_THREADS * 8u;
  c->total = o;
  return o <= 227u * 1024u;
}

template <int N, bool M, bool W, bool XF>
static int launch_variant(const ChunkArgs& a, const TcCfg& cfg, int grid, cudaStream_t s) {
  auto kern = tc_chunk_kernel<N, M, W, XF>;
  BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.total));
  kern<<<grid, TC_THREADS, cfg.total, s>>>(a, cfg);
  return 0;
}
template <bool M, bool W, bool XF>
static int launch_n(const ChunkArgs& a, const TcCfg& cfg, int grid, cudaStream_t s) {
  switch (wg::mma_n(cfg.NP)) {
    case 16: return launch_variant<16, M, W, XF>(a, cfg, grid, s);
    case 32: return launch_variant<32, M, W, XF>(a, cfg, grid, s);
    case 64: return launch_variant<64, M, W, XF>(a, cfg, grid, s);
    case 128: return launch_variant<128, M, W, XF>(a, cfg, grid, s);
    default: return launch_variant<256, M, W, XF>(a, cfg, grid, s);
  }
}

static int tc_grid(long long n, int sm_count) {
  const long long ntiles = (n + TBM - 1) / TBM;
  int grid = (int)(ntiles < sm_count ? ntiles : sm_count);
  return grid < 1 ? 1 : grid;
}

int launch_tc(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || (a.ldx % 4)) return BKM_EALIGN;
  const bool want_dist = a.min_out != nullptr || a.want_sum;
  TcCfg cfg;
  if (!make_cfg(a.d, a.k, mstep, &cfg)) return BKM_EUNSUPPORTED;
  const int grid = tc_grid(a.n, sm_count);
  *grid_out = grid;
  BKM_CUDA_TRY(cudaMemsetAsync(a.defer_cnt, 0, sizeof(int), s));
  int rc;
  if (mstep) rc = want_dist ? launch_n<true, true, false>(a, cfg, grid, s) : launch_n<true, false, false>(a, cfg, grid, s);
  else rc = want_dist ? launch_n<false, true, false>(a, cfg, grid, s) : launch_n<false, false, false>(a, cfg, grid, s);
  if (rc) return rc;
  note_launch(2);
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// (rows x k) block of distances / kernel values on the tensor path: same kernel, transform epilogue
int launch_tc_transform(const ChunkArgs& a, int sm_count, cudaStream_t s) {
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || (a.ldx % 4)) return BKM_EALIGN;
  TcCfg cfg;
  if (!make_cfg(a.d, a.k, false, &cfg)) return BKM_EUNSUPPORTED;
  const int rc = launch_n<false, false, true>(a, cfg, tc_grid(a.n, sm_count), s);
  if (rc) return rc;
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace bkm

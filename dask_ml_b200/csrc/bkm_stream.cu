// bkm_stream.cu — bandwidth-class fused E+M chunk kernel for tiny k*d (fp32, d <= 16, k <= 32): BASELINE config C4
// (120M x 13, k = 20; benchmarks/kmeans_airline.py shape) and the small plumbing shapes.
//
// The shape is HBM-bound (52..64 B per row, 2*d*k = 520 flops): the kernel is organised around the row stream.
//   * every WARP owns a private ring of SNSTG stages of 32 rows and keeps it full with 1-D bulk async copies
//     (cp.async.bulk global -> shared, completion on a per-stage mbarrier, issued by lane 0): no CTA-wide barrier in
//     the main loop, HBM requests stay in flight while the warp computes;
//   * E-step (sklearn pairwise_distances_argmin_min per chunk, dask_ml/metrics/pairwise.py:35-38): thread = row, the row
//     in registers, centres in shared memory as PAIRS {-2 c_2p, -2 c_2p+1} per feature so that one 64-bit load feeds
//     two distances (ptx::ffma2: two FFMA on sm_90); all k distances stay in registers, the arg-min and the near-tie test are
//     decoded from one FSET+FFMA per distance (same scheme as the tensor-path epilogue);
//   * rows whose best/second margin is inside the fp32 rounding bound are re-decided by the SAME thread in float64
//     against the float64 centres (rare: the warp diverges for them only);
//   * M-step (_centers_dense, dask_ml/cluster/k_means.py:572-582): lane j owns cluster j and adds the rows of its
//     warp's tile that carry label j into register-resident sums (k ballots per tile, no atomics, fixed order);
//     per-warp sums are folded in warp order into the CTA's partial at the end -> reduce_partials (float64, CTA order).
#include "bkm_common.cuh"
#include "bkm_ptx.cuh"
#include <math_constants.h>
#include <stdlib.h>

namespace bkm {

using namespace ptx;

static const int SW = 8;        // warps per CTA
static const int SNSTG = 4;     // ring stages per warp (32 rows each)

struct StreamSmem {
  uint32_t off_cp, off_cn, off_sums, off_cnt, off_red, off_bar, off_slot, off_ring, stage_bytes, total;
};

static inline StreamSmem stream_smem(int k, int d, long long ldx, int kpt, int dp) {
  StreamSmem S;
  uint32_t o = 0;
  S.off_cp = o;   o += (uint32_t)kpt * dp * 8;            // [kpt][dp] float2 {-2 c_2p,i , -2 c_2p+1,i}
  S.off_cn = o;   o += (uint32_t)kpt * 8;                 // [kpt] float2 {||c_2p||^2, ||c_2p+1||^2}
  o = (uint32_t)align_up(o, 16);
  S.off_sums = o; o += (uint32_t)k * d * 4;
  o = (uint32_t)align_up(o, 16);
  S.off_cnt = o;  o += (uint32_t)k * 4;
  o = (uint32_t)align_up(o, 16);
  S.off_red = o;  o += SW * 8;
  S.off_bar = o;  o += SW * SNSTG * 8;
  S.off_slot = o; o += SW * 32 * 4;                       // per warp: row mask of every cluster of the current tile
  o = (uint32_t)align_up(o, 128);
  S.stage_bytes = (uint32_t)(32 * ldx * 4);               // a multiple of 128
  S.off_ring = o; o += (uint32_t)SW * SNSTG * S.stage_bytes;
  S.total = o;
  return S;
}

// DH >= ceil(d / 2) feature pairs; KPT = number of centre pairs rounded up to an even number (k <= 4, 8, ..., 32).
// Both are compile-time so that the distance loop is branch-free straight-line FFMA code.
template <int DH, int KPT, bool MSTEP>
__global__ void __launch_bounds__(SW * 32, 2)
stream_chunk_kernel(ChunkArgs a, StreamSmem S) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  constexpr int DP = DH * 2;
  constexpr int D4 = (DP + 3) / 4;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d, k = a.k;
  const int L = (int)a.ldx;
  unsigned long long* cp = reinterpret_cast<unsigned long long*>(smem + S.off_cp);
  unsigned long long* cn2 = reinterpret_cast<unsigned long long*>(smem + S.off_cn);
  float* sums_s = reinterpret_cast<float*>(smem + S.off_sums);
  int* cnts_s = reinterpret_cast<int*>(smem + S.off_cnt);
  double* red_s = reinterpret_cast<double*>(smem + S.off_red);

  const float* gC = reinterpret_cast<const float*>(a.pack + a.L.off_cT);      // [k][d4] fp32, zero padded
  const int d4 = a.L.d4;
  const float* gCn = reinterpret_cast<const float*>(a.pack + a.L.off_cnT);    // [k]
  const double* gC64 = reinterpret_cast<const double*>(a.pack + a.L.off_c64); // [k][d]
  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const float* X = reinterpret_cast<const float*>(a.X);

  // ---- one-time staging: centre pairs, norms, zeroed CTA partials ----
  for (int i = tid; i < KPT * DP; i += SW * 32) {
    const int p = i / DP, f = i - p * DP;
    const int j0 = 2 * p, j1 = 2 * p + 1;
    const float v0 = (j0 < k && f < d) ? -2.f * gC[(size_t)j0 * d4 + f] : 0.f;
    const float v1 = (j1 < k && f < d) ? -2.f * gC[(size_t)j1 * d4 + f] : 0.f;
    cp[i] = pack2(v0, v1);
  }
  for (int p = tid; p < KPT; p += SW * 32)
    cn2[p] = pack2(2 * p < k ? gCn[2 * p] : CUDART_INF_F, 2 * p + 1 < k ? gCn[2 * p + 1] : CUDART_INF_F);
  if (MSTEP) {
    for (int i = tid; i < k * d; i += SW * 32) sums_s[i] = 0.f;
    for (int i = tid; i < k; i += SW * 32) cnts_s[i] = 0;
  }
  const float cnmax = (float)hdr->cn_max;

  // ---- the warp's private ring ----
  unsigned char* ring = smem + S.off_ring + (size_t)warp * SNSTG * S.stage_bytes;
  const uint32_t ring_u = smem_u32(ring);
  const uint32_t bar0 = smem_u32(smem + S.off_bar) + (uint32_t)warp * SNSTG * 8u;
  if (lane == 0) {
    for (int s = 0; s < SNSTG; ++s) mbar_init(bar0 + 8u * s, 1);
    mbar_fence_init();
  }
  __syncthreads();

  const long long ntiles = (a.n + 31) >> 5;
  const long long gw = (long long)blockIdx.x * SW + warp, nw = (long long)gridDim.x * SW;
  const uint32_t stage_bytes = S.stage_bytes;
  // Tiles before the last one are whole 32-row blocks [32 t, 32 t + 32) x ldx floats: one bulk copy each.  The last
  // tile of the chunk (partial, or ending at the last valid element of a padded view) is copied with plain loads.
  if (lane == 0) {
#pragma unroll 1
    for (int s = 0; s < SNSTG; ++s) {
      const long long t = gw + (long long)s * nw;
      if (t < ntiles - 1) {
        mbar_expect_tx(bar0 + 8u * s, stage_bytes);
        bulk_g2s(ring_u + (uint32_t)s * stage_bytes, X + t * 32 * (long long)L, stage_bytes, bar0 + 8u * s);
      }
    }
  }

  float macc[MSTEP ? DP : 1];
#pragma unroll
  for (int i = 0; i < (MSTEP ? DP : 1); ++i) macc[i] = 0.f;
  int mcnt = 0;
  double dsum = 0.0;
  const bool want_dist = a.want_sum || a.min_out != nullptr;

  long long it = 0;
#pragma unroll 1
  for (long long t = gw; t < ntiles; t += nw, ++it) {
    const int s = (int)(it % SNSTG);
    float* xs = reinterpret_cast<float*>(ring + (size_t)s * stage_bytes);
    const long long r0 = t << 5;
    const int rows = (int)min(32LL, a.n - r0);
    if (t == ntiles - 1) {
      const int nel = (rows - 1) * L + d;
      const float* src = X + r0 * (long long)L;
      for (int e = lane; e < nel; e += 32) xs[e] = src[e];
      __syncwarp();
    } else {
      mbar_wait(bar0 + 8u * s, (uint32_t)((it / SNSTG) & 1));
    }
    const bool valid = lane < rows;

    // ---- the row, in registers ----
    float x[DP];
    {
      const float* xr = xs + lane * L;
      if ((L & 3) == 0) {
#pragma unroll
        for (int q = 0; q < D4; ++q) {
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (valid && q * 4 < d) v = *reinterpret_cast<const float4*>(xr + q * 4);
          x[q * 4 + 0] = v.x;
          if (q * 4 + 1 < DP) x[q * 4 + 1] = q * 4 + 1 < d ? v.y : 0.f;
          if (q * 4 + 2 < DP) x[q * 4 + 2] = q * 4 + 2 < d ? v.z : 0.f;
          if (q * 4 + 3 < DP) x[q * 4 + 3] = q * 4 + 3 < d ? v.w : 0.f;
        }
      } else {
#pragma unroll
        for (int i = 0; i < DP; ++i) x[i] = (valid && i < d) ? xr[i] : 0.f;
      }
    }
    float xn = 0.f;
#pragma unroll
    for (int i = 0; i < DP; ++i) xn = fmaf(x[i], x[i], xn);

    // ---- E-step: all k distances (GEMM form ||c||^2 - 2 x.c), two per ffma2 ----
    unsigned long long dp[KPT];
#pragma unroll
    for (int g = 0; g + 4 <= KPT; g += 4) {
      unsigned long long a0 = cn2[g], a1 = cn2[g + 1], a2 = cn2[g + 2], a3 = cn2[g + 3];
#pragma unroll
      for (int i = 0; i < DP; i += 2) {
        // {x_i, x_i}: the scalar as both halves of the pair
        const unsigned long long x0 = pack2(x[i], x[i]), x1 = pack2(x[i + 1], x[i + 1]);
        const ulonglong2 c0 = *reinterpret_cast<const ulonglong2*>(cp + (g + 0) * DP + i);
        const ulonglong2 c1 = *reinterpret_cast<const ulonglong2*>(cp + (g + 1) * DP + i);
        const ulonglong2 c2 = *reinterpret_cast<const ulonglong2*>(cp + (g + 2) * DP + i);
        const ulonglong2 c3 = *reinterpret_cast<const ulonglong2*>(cp + (g + 3) * DP + i);
        a0 = ffma2(x0, c0.x, a0); a1 = ffma2(x0, c1.x, a1); a2 = ffma2(x0, c2.x, a2); a3 = ffma2(x0, c3.x, a3);
        a0 = ffma2(x1, c0.y, a0); a1 = ffma2(x1, c1.y, a1); a2 = ffma2(x1, c2.y, a2); a3 = ffma2(x1, c3.y, a3);
      }
      dp[g] = a0; dp[g + 1] = a1; dp[g + 2] = a2; dp[g + 3] = a3;
    }
    if (KPT & 2) {                                        // compile-time tail: two more pairs
      constexpr int g = KPT & ~3;
      unsigned long long a0 = cn2[g], a1 = cn2[g + 1];
#pragma unroll
      for (int i = 0; i < DP; i += 2) {
        const unsigned long long x0 = pack2(x[i], x[i]), x1 = pack2(x[i + 1], x[i + 1]);
        const ulonglong2 c0 = *reinterpret_cast<const ulonglong2*>(cp + (g + 0) * DP + i);
        const ulonglong2 c1 = *reinterpret_cast<const ulonglong2*>(cp + (g + 1) * DP + i);
        a0 = ffma2(x0, c0.x, a0); a1 = ffma2(x0, c1.x, a1);
        a0 = ffma2(x1, c0.y, a0); a1 = ffma2(x1, c1.y, a1);
      }
      dp[g] = a0; dp[g + 1] = a1;
    }
    // minimum, then one FSET + FFMA per distance: every distance within `bound` of the minimum adds 1 + j/1024;
    // exactly one hit decodes the arg-min, two or more mark a near-tie
    float m1 = CUDART_INF_F;
#pragma unroll
    for (int p = 0; p < KPT; ++p) {
      float lo, hi;
      unpack2(dp[p], lo, hi);
      m1 = fmin3(m1, lo, hi);
    }
    const float bound = a.tau * (xn + cnmax);
    const float thr = m1 + bound;
    float h0 = 0.f, h1 = 0.f;
#pragma unroll
    for (int p = 0; p < KPT; ++p) {
      float lo, hi;
      unpack2(dp[p], lo, hi);
      h0 = fmaf(fset_le(lo, thr), 1.f + (float)(2 * p) * 0.0009765625f, h0);
      h1 = fmaf(fset_le(hi, thr), 1.f + (float)(2 * p + 1) * 0.0009765625f, h1);
    }
    const float hits = h0 + h1;
    int bj = (int)((hits - 1.f) * 1024.f + 0.5f);
    double d2x = -1.0;                                    // exact float64 distance when the row took the float64 path
    if (valid && !(hits >= 1.f && hits < 2.f) && k > 1) {
      if (a.tau > 0.f) {
        // near-tie (or non-finite): decide in float64 against the float64 centres, lowest index on exact ties
        double bd = CUDART_INF;
        bj = 0;
        for (int j = 0; j < k; ++j) {
          const double* c = gC64 + (size_t)j * d;
          double sacc = 0.0;
#pragma unroll
          for (int i = 0; i < DP; ++i)
            if (i < d) { const double df = (double)x[i] - c[i]; sacc = fma(df, df, sacc); }
          if (sacc < bd) { bd = sacc; bj = j; }
        }
        d2x = bd;
      } else {
        // re-check disabled (BKM_FLAG_NO_RECHECK): first index that attains the fp32 minimum
        bj = 0;
        bool found = false;
#pragma unroll
        for (int p = 0; p < KPT; ++p) {
          float lo, hi;
          unpack2(dp[p], lo, hi);
          if (!found && lo == m1) { bj = 2 * p; found = true; }
          if (!found && hi == m1) { bj = 2 * p + 1; found = true; }
        }
      }
    }
    if (k == 1) bj = 0;
    if (!valid) bj = -1;

    // ---- outputs of the E-step ----
    if (valid) {
      if (a.labels) a.labels[r0 + lane] = bj;
      if (want_dist) {
        double dd = d2x;
        if (dd < 0.0) {
          // winning distance in direct form sum (x - c)^2 (no cancellation); c = -0.5 * the staged pair entry
          const float* cw = reinterpret_cast<const float*>(cp + (size_t)(bj >> 1) * DP) + (bj & 1);
          float sacc = 0.f;
#pragma unroll
          for (int i = 0; i < DP; ++i)
            if (i < d) { const float df = fmaf(0.5f, cw[2 * i], x[i]); sacc = fmaf(df, df, sacc); }
          dd = (double)sacc;
        }
        const double outv = a.squared ? dd : sqrt(dd);
        dsum += outv;
        if (a.min_out) reinterpret_cast<float*>(a.min_out)[r0 + lane] = (float)outv;
      }
    }

    // ---- M-step: lane j takes the rows of this tile labelled j ----
    if (MSTEP) {
      // row mask of every cluster: lanes with the same label hold the same match mask and post it to the slot
      // of their cluster (identical values: the colliding stores are benign), the owner lane picks it up
      unsigned* slot = reinterpret_cast<unsigned*>(smem + S.off_slot) + warp * 32;
      slot[lane] = 0u;
      const unsigned same = __match_any_sync(0xffffffffu, bj);
      __syncwarp();
      if (bj >= 0) slot[bj] = same;
      __syncwarp();
      unsigned mine = slot[lane];
      mcnt += __popc(mine);
#pragma unroll 1
      while (__any_sync(0xffffffffu, mine != 0)) {
        if (mine) {
          const int b = __ffs(mine) - 1;
          mine &= mine - 1;
          const float* xr = xs + b * L;
#pragma unroll
          for (int i = 0; i < (MSTEP ? DP : 1); ++i)
            if (i < d) macc[i] += xr[i];
        }
      }
    }

    // ---- refill this stage ----
    __syncwarp();
    if (lane == 0) {
      const long long tn = t + (long long)SNSTG * nw;
      if (tn < ntiles - 1) {
        mbar_expect_tx(bar0 + 8u * s, stage_bytes);
        bulk_g2s(ring_u + (uint32_t)s * stage_bytes, X + tn * 32 * (long long)L, stage_bytes, bar0 + 8u * s);
      }
    }
  }

  // ---- fold the warps' register sums into the CTA partial, in warp order (reproducible) ----
  if (MSTEP) {
    for (int w = 0; w < SW; ++w) {
      if (warp == w && lane < k) {
#pragma unroll
        for (int i = 0; i < (MSTEP ? DP : 1); ++i)
          if (i < d) sums_s[lane * d + i] += macc[i];
        cnts_s[lane] += mcnt;
      }
      __syncthreads();
    }
    float* g = reinterpret_cast<float*>(a.psum) + (size_t)blockIdx.x * k * d;
    for (int i = tid; i < k * d; i += SW * 32) g[i] = sums_s[i];
    int* gc = a.pcnt + (size_t)blockIdx.x * k;
    for (int i = tid; i < k; i += SW * 32) gc[i] = cnts_s[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
  if (lane == 0) red_s[warp] = dsum;
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0;
    for (int w = 0; w < SW; ++w) sacc += red_s[w];
    a.pin[blockIdx.x] = sacc;
  }
}

// ==========================================================================================================
// Two rows per thread (k <= 24): the ffma2 pair is {row l, row l + 32} of a 64-row warp tile against ONE centre value
// (broadcast operand), so every centre load (LDS.128 of four features) feeds two rows, the per-tile overheads (ring
// refill, label masks, M-step loop) are paid once per 64 rows and the lane-owns-cluster M-step sees twice the rows per
// cluster and pass (better lane utilisation: its trip count is the LARGEST list of the tile).
// ==========================================================================================================
static const int S2_NSTG = 3;       // ring stages per warp (64 rows each)

struct Stream2Smem {
  uint32_t off_c, off_cn, off_cnt, off_red, off_bar, off_slot, off_lab, off_wsum, off_ring, stage_bytes, total;
};
static inline Stream2Smem stream2_smem(int k, int d, long long ldx, int kc, int dp) {
  Stream2Smem S;
  uint32_t o = 0;
  S.off_c = o;    o += (uint32_t)kc * dp * 4;             // [kc][dp] floats: -2 c (zero padded)
  S.off_cn = o;   o += (uint32_t)kc * 4;                  // [kc] ||c||^2 (+inf for j >= k)
  o = (uint32_t)align_up(o, 16);
  S.off_cnt = o;  o += (uint32_t)k * 4;
  o = (uint32_t)align_up(o, 16);
  S.off_red = o;  o += SW * 8;
  S.off_bar = o;  o += SW * S2_NSTG * 8;
  S.off_slot = o; o += SW * 64 * 4;                       // per warp: two row masks per cluster
  S.off_lab = o;  o += SW * 64 * 4;                       // per warp: the tile's labels (invalid rows -> kc, a trash slot)
  o = (uint32_t)align_up(o, 128);
  S.off_wsum = o; o += (uint32_t)SW * (kc + 1) * 32 * 4;  // per warp: [kc + 1][2 row halves][16 features] running sums
  o = (uint32_t)align_up(o, 128);
  S.stage_bytes = (uint32_t)(64 * ldx * 4);
  S.off_ring = o; o += (uint32_t)SW * S2_NSTG * S.stage_bytes + 128;      // + slack: the M-step reads whole DP-float rows
  S.total = o;
  return S;
}

// M-step of one 64-row tile: lane (f = lane & 15, h = lane >> 4) adds feature f of 32 rows into the warp's private
// shared-memory sums [label][h][f] (plain load / add / store: each address belongs to one lane, and the two halves of
// the warp have their own copies, so there is no race and the order is fixed).  The trip count does not depend on how
// the rows are spread over the clusters (the lane-owns-cluster walk ran for the LONGEST list of the tile: 12 of 64
// rows on the airline-shaped data).  Half h takes rows r0(i) + h * S, S chosen from the row pitch so that the two
// halves read different banks (S * L = 16 mod 32 when L has fewer than 5 trailing zero bits).
template <int S>
__device__ __forceinline__ void stream2_mstep_tile(const float* xs_lane, const int* lab_h, float* ws, int L) {
#pragma unroll
  for (int b = 0; b < 32; b += 8) {
    int l[8];
    float x[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r0 = (((b + i) & ~(S - 1)) << 1) + ((b + i) & (S - 1));
      l[i] = lab_h[r0];
      x[i] = xs_lane[r0 * L];
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) ws[l[i] * 32] += x[i];
  }
}

// DH = feature pairs (DP = 2 DH >= d), KC = centres rounded up to a multiple of 4 (<= 24)
template <int DH, int KC, bool MSTEP>
__global__ void __launch_bounds__(SW * 32, 2)
stream2_chunk_kernel(ChunkArgs a, Stream2Smem S) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  constexpr int DP = DH * 2;
  constexpr int D4 = (DP + 3) / 4;
  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d, k = a.k;
  const int L = (int)a.ldx;
  float* cs = reinterpret_cast<float*>(smem + S.off_c);
  float* cns = reinterpret_cast<float*>(smem + S.off_cn);
  int* cnts_s = reinterpret_cast<int*>(smem + S.off_cnt);
  double* red_s = reinterpret_cast<double*>(smem + S.off_red);
  const float* gC = reinterpret_cast<const float*>(a.pack + a.L.off_cT);      // [k][d4] fp32, zero padded
  const int d4 = a.L.d4;
  const float* gCn = reinterpret_cast<const float*>(a.pack + a.L.off_cnT);
  const double* gC64 = reinterpret_cast<const double*>(a.pack + a.L.off_c64);
  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const float* X = reinterpret_cast<const float*>(a.X);

  constexpr int CP = D4 * 4;                               // centre row pitch in shared memory (16-byte rows)
  for (int i = tid; i < KC * CP; i += SW * 32) {
    const int j = i / CP, f = i - j * CP;
    cs[i] = (j < k && f < d) ? -2.f * gC[(size_t)j * d4 + f] : 0.f;
  }
  for (int j = tid; j < KC; j += SW * 32) cns[j] = j < k ? gCn[j] : CUDART_INF_F;
  float* wsum = reinterpret_cast<float*>(smem + S.off_wsum);               // [SW][KC + 1][2][16]
  if (MSTEP) {
    for (int i = tid; i < k; i += SW * 32) cnts_s[i] = 0;
    for (int i = tid; i < SW * (KC + 1) * 32; i += SW * 32) wsum[i] = 0.f;
  }
  const float cnmax = (float)hdr->cn_max;

  unsigned char* ring = smem + S.off_ring + (size_t)warp * S2_NSTG * S.stage_bytes;
  const uint32_t ring_u = smem_u32(ring);
  const uint32_t bar0 = smem_u32(smem + S.off_bar) + (uint32_t)warp * S2_NSTG * 8u;
  if (lane == 0) {
    for (int s = 0; s < S2_NSTG; ++s) mbar_init(bar0 + 8u * s, 1);
    mbar_fence_init();
  }
  __syncthreads();

  const long long ntiles = (a.n + 63) >> 6;
  const long long gw = (long long)blockIdx.x * SW + warp, nw = (long long)gridDim.x * SW;
  const uint32_t stage_bytes = S.stage_bytes;
  if (lane == 0) {
#pragma unroll 1
    for (int s = 0; s < S2_NSTG; ++s) {
      const long long t = gw + (long long)s * nw;
      if (t < ntiles - 1) {
        mbar_expect_tx(bar0 + 8u * s, stage_bytes);
        bulk_g2s(ring_u + (uint32_t)s * stage_bytes, X + t * 64 * (long long)L, stage_bytes, bar0 + 8u * s);
      }
    }
  }

  int mcnt = 0;
  // pairing of the two half-warps' rows (see stream2_mstep_tile)
  const int tzL = __ffs(L) - 1;
  const int msS = tzL >= 4 ? 1 : (16 >> tzL);
  const int mf = lane & 15, mh = lane >> 4;
  int* lab_w = reinterpret_cast<int*>(smem + S.off_lab) + warp * 64;
  float* ws_lane = wsum + (size_t)warp * (KC + 1) * 32 + mh * 16 + mf;
  double dsum = 0.0;
  const bool want_dist = a.want_sum || a.min_out != nullptr;

  long long it = 0;
#pragma unroll 1
  for (long long t = gw; t < ntiles; t += nw, ++it) {
    const int s = (int)(it % S2_NSTG);
    float* xs = reinterpret_cast<float*>(ring + (size_t)s * stage_bytes);
    const long long r0 = t << 6;
    const int rows = (int)min(64LL, a.n - r0);
    if (t == ntiles - 1) {
      const int nel = (rows - 1) * L + d;
      const float* src = X + r0 * (long long)L;
      for (int e = lane; e < nel; e += 32) xs[e] = src[e];
      __syncwarp();
    } else {
      mbar_wait(bar0 + 8u * s, (uint32_t)((it / S2_NSTG) & 1));
    }
    const bool v0 = lane < rows, v1 = lane + 32 < rows;

    // ---- two rows per thread, packed per feature: xp[i] = {x_i of row lane, x_i of row lane + 32} ----
    unsigned long long xp[DP];
    float xn0 = 0.f, xn1 = 0.f;
    {
      const float* xa = xs + lane * L;
      const float* xb = xs + (lane + 32) * L;
      if ((L & 3) == 0) {
#pragma unroll
        for (int q = 0; q < D4; ++q) {
          float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
          if (v0 && q * 4 < d) va = *reinterpret_cast<const float4*>(xa + q * 4);
          if (v1 && q * 4 < d) vb = *reinterpret_cast<const float4*>(xb + q * 4);
          const float fa[4] = {va.x, va.y, va.z, va.w}, fb[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (q * 4 + e < DP) {
              const float ea = q * 4 + e < d ? fa[e] : 0.f, eb = q * 4 + e < d ? fb[e] : 0.f;
              xp[q * 4 + e] = pack2(ea, eb);
              xn0 = fmaf(ea, ea, xn0); xn1 = fmaf(eb, eb, xn1);
            }
        }
      } else {
#pragma unroll
        for (int i = 0; i < DP; ++i) {
          const float ea = (v0 && i < d) ? xa[i] : 0.f, eb = (v1 && i < d) ? xb[i] : 0.f;
          xp[i] = pack2(ea, eb);
          xn0 = fmaf(ea, ea, xn0); xn1 = fmaf(eb, eb, xn1);
        }
      }
    }

    // ---- E-step: dist pair {row0, row1} per centre ----
    unsigned long long dp[KC];
#pragma unroll
    for (int g = 0; g < KC; g += 4) {
      const float4 cnv = *reinterpret_cast<const float4*>(cns + g);
      unsigned long long a0 = pack2(cnv.x, cnv.x), a1 = pack2(cnv.y, cnv.y), a2 = pack2(cnv.z, cnv.z), a3 = pack2(cnv.w, cnv.w);
#pragma unroll
      for (int q = 0; q < D4; ++q) {
        const float4 c0 = *reinterpret_cast<const float4*>(cs + (g + 0) * CP + q * 4);
        const float4 c1 = *reinterpret_cast<const float4*>(cs + (g + 1) * CP + q * 4);
        const float4 c2 = *reinterpret_cast<const float4*>(cs + (g + 2) * CP + q * 4);
        const float4 c3 = *reinterpret_cast<const float4*>(cs + (g + 3) * CP + q * 4);
        const float f0[4] = {c0.x, c0.y, c0.z, c0.w}, f1[4] = {c1.x, c1.y, c1.z, c1.w};
        const float f2[4] = {c2.x, c2.y, c2.z, c2.w}, f3[4] = {c3.x, c3.y, c3.z, c3.w};
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (q * 4 + e < DP) {
            const unsigned long long xv = xp[q * 4 + e];
            a0 = ffma2(xv, pack2(f0[e], f0[e]), a0); a1 = ffma2(xv, pack2(f1[e], f1[e]), a1);
            a2 = ffma2(xv, pack2(f2[e], f2[e]), a2); a3 = ffma2(xv, pack2(f3[e], f3[e]), a3);
          }
      }
      dp[g] = a0; dp[g + 1] = a1; dp[g + 2] = a2; dp[g + 3] = a3;
    }
    // ---- decode both rows: minimum, then FSET + FFMA per distance (see the one-row kernel) ----
    int bjr[2];
    double d2x[2] = {-1.0, -1.0};
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float m1 = CUDART_INF_F;
#pragma unroll
      for (int j = 0; j + 1 < KC; j += 2) {
        float lo0, hi0, lo1, hi1;
        unpack2(dp[j], lo0, hi0); unpack2(dp[j + 1], lo1, hi1);
        m1 = fmin3(m1, h ? hi0 : lo0, h ? hi1 : lo1);
      }
      const float xn = h ? xn1 : xn0;
      const float thr = m1 + a.tau * (xn + cnmax);
      float h0 = 0.f, h1 = 0.f;
#pragma unroll
      for (int j = 0; j + 1 < KC; j += 2) {
        float lo0, hi0, lo1, hi1;
        unpack2(dp[j], lo0, hi0); unpack2(dp[j + 1], lo1, hi1);
        h0 = fmaf(fset_le(h ? hi0 : lo0, thr), 1.f + (float)j * 0.0009765625f, h0);
        h1 = fmaf(fset_le(h ? hi1 : lo1, thr), 1.f + (float)(j + 1) * 0.0009765625f, h1);
      }
      const float hits = h0 + h1;
      int bj = (int)((hits - 1.f) * 1024.f + 0.5f);
      const bool valid = h ? v1 : v0;
      if (valid && !(hits >= 1.f && hits < 2.f) && k > 1) {
        if (a.tau > 0.f) {
          double bd = CUDART_INF;
          bj = 0;
          for (int j = 0; j < k; ++j) {
            const double* c = gC64 + (size_t)j * d;
            double sacc = 0.0;
#pragma unroll
            for (int i = 0; i < DP; ++i)
              if (i < d) {
                float ea, eb;
                unpack2(xp[i], ea, eb);
                const double df = (double)(h ? eb : ea) - c[i];
                sacc = fma(df, df, sacc);
              }
            if (sacc < bd) { bd = sacc; bj = j; }
          }
          d2x[h] = bd;
        } else {
          bj = 0;
          bool found = false;
#pragma unroll
          for (int j = 0; j < KC; ++j) {
            float lo, hi;
            unpack2(dp[j], lo, hi);
            if (!found && (h ? hi : lo) == m1) { bj = j; found = true; }
          }
        }
      }
      if (k == 1) bj = 0;
      if (!valid) bj = -1;
      bjr[h] = bj;
      if (valid) {
        const long long row = r0 + lane + 32 * h;
        if (a.labels) a.labels[row] = bj;
        if (want_dist) {
          double dd = d2x[h];
          if (dd < 0.0) {
            const float* cw = cs + (size_t)bj * CP;
            float sacc = 0.f;
#pragma unroll
            for (int i = 0; i < DP; ++i)
              if (i < d) {
                float ea, eb;
                unpack2(xp[i], ea, eb);
                const float df = fmaf(0.5f, cw[i], h ? eb : ea);
                sacc = fmaf(df, df, sacc);
              }
            dd = (double)sacc;
          }
          const double outv = a.squared ? dd : sqrt(dd);
          dsum += outv;
          if (a.min_out) reinterpret_cast<float*>(a.min_out)[row] = (float)outv;
        }
      }
    }

    // ---- M-step: counts per cluster from the label masks, sums through the per-warp shared-memory accumulators ----
    if (MSTEP) {
      unsigned* slot = reinterpret_cast<unsigned*>(smem + S.off_slot) + warp * 64;
      slot[lane] = 0u; slot[32 + lane] = 0u;
      lab_w[lane] = bjr[0] >= 0 ? bjr[0] : KC;
      lab_w[32 + lane] = bjr[1] >= 0 ? bjr[1] : KC;
      const unsigned same0 = __match_any_sync(0xffffffffu, bjr[0]);
      const unsigned same1 = __match_any_sync(0xffffffffu, bjr[1]);
      __syncwarp();
      if (bjr[0] >= 0) slot[bjr[0]] = same0;
      if (bjr[1] >= 0) slot[32 + bjr[1]] = same1;
      __syncwarp();
      mcnt += __popc(slot[lane]) + __popc(slot[32 + lane]);
      const float* xl = xs + mh * msS * L + mf;
      const int* lh = lab_w + mh * msS;
      switch (msS) {
        case 16: stream2_mstep_tile<16>(xl, lh, ws_lane, L); break;
        case 8: stream2_mstep_tile<8>(xl, lh, ws_lane, L); break;
        case 4: stream2_mstep_tile<4>(xl, lh, ws_lane, L); break;
        case 2: stream2_mstep_tile<2>(xl, lh, ws_lane, L); break;
        default: stream2_mstep_tile<1>(xl, lh, ws_lane, L); break;
      }
    }

    // ---- refill this stage ----
    __syncwarp();
    if (lane == 0) {
      const long long tn = t + (long long)S2_NSTG * nw;
      if (tn < ntiles - 1) {
        mbar_expect_tx(bar0 + 8u * s, stage_bytes);
        bulk_g2s(ring_u + (uint32_t)s * stage_bytes, X + tn * 64 * (long long)L, stage_bytes, bar0 + 8u * s);
      }
    }
  }

  if (MSTEP) {
    for (int w = 0; w < SW; ++w) {
      if (warp == w && lane < k) cnts_s[lane] += mcnt;
      __syncthreads();
    }
    // per-CTA partial: the 2 * SW accumulators of (cluster, feature) added in a fixed order
    float* g = reinterpret_cast<float*>(a.psum) + (size_t)blockIdx.x * k * d;
    for (int i = tid; i < k * d; i += SW * 32) {
      const int j = i / d, f = i - j * d;
      float sacc = 0.f;
      for (int w = 0; w < SW; ++w) {
        const float* p = wsum + ((size_t)w * (KC + 1) + j) * 32 + f;
        sacc += p[0];
        sacc += p[16];
      }
      g[i] = sacc;
    }
    int* gc = a.pcnt + (size_t)blockIdx.x * k;
    for (int i = tid; i < k; i += SW * 32) gc[i] = cnts_s[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
  if (lane == 0) red_s[warp] = dsum;
  __syncthreads();
  if (tid == 0) {
    double sacc = 0.0;
    for (int w = 0; w < SW; ++w) sacc += red_s[w];
    a.pin[blockIdx.x] = sacc;
  }
}

template <int DH, int KC>
static int launch_stream2_dk(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  Stream2Smem S = stream2_smem(a.k, a.d, a.ldx, KC, (2 * DH + 3) / 4 * 4);
  if (S.total > 227 * 1024) return BKM_EUNSUPPORTED;
  const long long ntiles = (a.n + 63) / 64;
  int occ = 0;
#define STREAM2_GO(M)                                                                                       \
  {                                                                                                         \
    auto kern = stream2_chunk_kernel<DH, KC, M>;                                                            \
    BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S.total));    \
    BKM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, SW * 32, S.total));              \
    if (occ < 1) return BKM_EUNSUPPORTED;                                                                   \
    long long grid = (long long)sm_count * occ;                                                             \
    if (grid > a.psum_slots) grid = a.psum_slots;                                                           \
    if (grid > a.part_slots) grid = a.part_slots;                                                           \
    const long long need = (ntiles + SW - 1) / SW;                                                          \
    if (grid > need) grid = need;                                                                           \
    if (grid < 1) grid = 1;                                                                                 \
    *grid_out = (int)grid;                                                                                  \
    kern<<<(int)grid, SW * 32, S.total, s>>>(a, S);                                                         \
  }
  if (mstep) STREAM2_GO(true) else STREAM2_GO(false)
#undef STREAM2_GO
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

template <int DH>
static int launch_stream2_d(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  switch ((a.k + 3) / 4) {
    case 1: return launch_stream2_dk<DH, 4>(a, mstep, sm_count, grid_out, s);
    case 2: return launch_stream2_dk<DH, 8>(a, mstep, sm_count, grid_out, s);
    case 3: return launch_stream2_dk<DH, 12>(a, mstep, sm_count, grid_out, s);
    case 4: return launch_stream2_dk<DH, 16>(a, mstep, sm_count, grid_out, s);
    case 5: return launch_stream2_dk<DH, 20>(a, mstep, sm_count, grid_out, s);
    default: return launch_stream2_dk<DH, 24>(a, mstep, sm_count, grid_out, s);
  }
}

bool stream_supported(int d, int k, int dtype) {
  return dtype == BKM_F32 && d >= 1 && d <= 16 && k >= 1 && k <= 32;
}

template <int DH, int KPT>
static int launch_stream_dk(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  StreamSmem S = stream_smem(a.k, a.d, a.ldx, KPT, 2 * DH);
  if (S.total > 227 * 1024) return BKM_EUNSUPPORTED;
  const long long ntiles = (a.n + 31) / 32;
  int occ = 0;
#define STREAM_GO(M)                                                                                        \
  {                                                                                                         \
    auto kern = stream_chunk_kernel<DH, KPT, M>;                                                            \
    BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)S.total));    \
    BKM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, SW * 32, S.total));              \
    if (occ < 1) return BKM_EUNSUPPORTED;                                                                   \
    long long grid = (long long)sm_count * occ;                                                             \
    if (grid > a.psum_slots) grid = a.psum_slots;                                                           \
    if (grid > a.part_slots) grid = a.part_slots;                                                           \
    const long long need = (ntiles + SW - 1) / SW;                                                          \
    if (grid > need) grid = need;                                                                           \
    if (grid < 1) grid = 1;                                                                                 \
    *grid_out = (int)grid;                                                                                  \
    kern<<<(int)grid, SW * 32, S.total, s>>>(a, S);                                                         \
  }
  if (mstep) STREAM_GO(true) else STREAM_GO(false)
#undef STREAM_GO
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

template <int DH>
static int launch_stream_d(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  switch ((a.k + 3) / 4) {                 // pairs, rounded up to an even count
    case 1: return launch_stream_dk<DH, 2>(a, mstep, sm_count, grid_out, s);
    case 2: return launch_stream_dk<DH, 4>(a, mstep, sm_count, grid_out, s);
    case 3: return launch_stream_dk<DH, 6>(a, mstep, sm_count, grid_out, s);
    case 4: return launch_stream_dk<DH, 8>(a, mstep, sm_count, grid_out, s);
    case 5: return launch_stream_dk<DH, 10>(a, mstep, sm_count, grid_out, s);
    case 6: return launch_stream_dk<DH, 12>(a, mstep, sm_count, grid_out, s);
    case 7: return launch_stream_dk<DH, 14>(a, mstep, sm_count, grid_out, s);
    default: return launch_stream_dk<DH, 16>(a, mstep, sm_count, grid_out, s);
  }
}

// BKM_EALIGN when the row block cannot be bulk-copied (the caller then falls back to the generic CUDA-core kernel).
int launch_stream(const ChunkArgs& a, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  if (!stream_supported(a.d, a.k, BKM_F32)) return BKM_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || a.ldx > 64) return BKM_EALIGN;
  if (a.k <= 24 && a.ldx <= 32 && !getenv("BKM_STREAM_V1")) {        // two rows per thread
    if (a.d <= 4) return launch_stream2_d<2>(a, mstep, sm_count, grid_out, s);
    if (a.d <= 8) return launch_stream2_d<4>(a, mstep, sm_count, grid_out, s);
    if (a.d <= 12) return launch_stream2_d<6>(a, mstep, sm_count, grid_out, s);
    if (a.d <= 14) return launch_stream2_d<7>(a, mstep, sm_count, grid_out, s);
    return launch_stream2_d<8>(a, mstep, sm_count, grid_out, s);
  }
  // feature pairs (compile-time): d <= 4, 8, 12, 14, 16
  if (a.d <= 4) return launch_stream_d<2>(a, mstep, sm_count, grid_out, s);
  if (a.d <= 8) return launch_stream_d<4>(a, mstep, sm_count, grid_out, s);
  if (a.d <= 12) return launch_stream_d<6>(a, mstep, sm_count, grid_out, s);
  if (a.d <= 14) return launch_stream_d<7>(a, mstep, sm_count, grid_out, s);
  return launch_stream_d<8>(a, mstep, sm_count, grid_out, s);
}

}  // namespace bkm

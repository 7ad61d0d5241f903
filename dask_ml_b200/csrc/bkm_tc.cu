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
// CTA = NWG warpgroups (1 CTA per SM): 3 in the M-step variants, 2 in the others (tc_warpgroups).  The CTA's tiles
// stream through a ring of S shared-memory slots filled by TMA (local tile lt -> slot lt % S, one "full" mbarrier per
// slot; fp32 rows in 32-column SWIZZLE_128B boxes, zero-filled beyond n and d by the copy engine).  Warpgroup w owns
// the CTA's tiles lt with lt % NWG == w and runs, per tile:
//   the wait for the tile's slot;
//   the fp16 (hi, lo) A fragments of s X built in registers (and ||s x||^2);
//   3 KS wgmma.m64nNk16 (KS = ceil(d/16), a template parameter so that they issue back to back) with B
//   (= -2 s C as fp16 hi / lo, SWIZZLE_128B K-major) resident in shared memory; N = 256 runs as two column halves of
//   128;
//   the arg-min epilogue from the register accumulators in two passes (the row minimum, then the count and index
//   of the columns within the near-tie bound of it), one column half at a time: half 1's MMAs reuse half 0's
//   accumulator registers once its passes are done (wg::near_tie_cols), so a thread keeps 64 of them, not 128;
//   the winning distance in direct form (x - c)^2 in fp32, and the M-step;
//   after the warpgroup's last read of the slot, the load of tile lt + S into it (no separate producer).
// The M-step adds the tile's rows in row order into the CTA's sums; the warpgroups take turns in tile order (named
// barriers), so every cluster's sum is formed in one fixed order and the sums are bit-reproducible.  Each sums element
// has one owning thread (feature pair f2, label class q = c % 4, warp q of its warpgroup); before its turn a warp lists
// the tile's rows of its class, so that the turn touches only owned rows, and marks the batches of 8 rows in which a
// label repeats (only those forward running sums).  The turn order is kept per warp triple: warp w of each warpgroup
// owns the same elements.  One warpgroup's MMAs overlap the others' epilogues / M-steps; the third warpgroup of the
// M-step variants gives each scheduler a third warp to issue from while the others wait on shared memory, barriers
// or the tensor cores.
#include "bkm_common.cuh"
#include "bkm_wgmma.cuh"
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <math_constants.h>

namespace bkm {

static const int TBM = 64;           // rows per warpgroup tile (wgmma M)
// Warpgroups of a CTA.  The M-step variants run three: at 384 threads a thread has 168 registers, which the arg-min by
// column halves leaves enough.  The others keep two: without the turn order, a slot has one reader only when S is a
// multiple of the warpgroup count (see place_ring), and their S = 8 is not a multiple of 3.
__host__ __device__ constexpr int tc_warpgroups(bool mstep) { return mstep ? 3 : 2; }
static const int TC_MAX_THREADS = 128 * tc_warpgroups(true);
// X ring: a slot holds one 64 x 64 fp32 tile as two TMA boxes of 32 columns (box b: columns 32b .. 32b + 31, 64 rows of
// 128 bytes, SWIZZLE_128B: 16-byte chunk q of row r sits at chunk q ^ (r & 7)), so that a warp's reads of 8 rows x one
// chunk, or of one row x 32 columns, hit 32 different banks
static const uint32_t XBOX_BYTES = TBM * 128u;
static const uint32_t XSLOT_BYTES = 2u * XBOX_BYTES;
static const int TC_MAX_STAGES = 8;
// two slots per warpgroup of the two-warpgroup variants (the tile being worked on and the next one); more slots than
// warpgroups for the three of the M-step variants (the slot-reuse argument at the wait in tc_chunk_kernel).  Every
// supported shape (d <= 64, k <= 256) leaves room for at least 4 (the M-step variants at N = 256: 5)
static const int TC_MIN_STAGES = 4;

struct TcCfg {
  int KS;        // MMA K-steps of 16 (ceil(d/16))
  int NP;        // padded centre count (multiple of 16, <= 256)
  int S;         // slots of the X ring
  uint32_t off_bhi, off_blo, off_sum, off_cn, off_cnt, off_lab, off_dp, off_cls, off_bar, off_ring, total;
};

// Epilogue of tc_chunk_kernel (all four share the MMAs, the tile pipeline and the A-fragment build):
//   ARGMIN  labels / M-step (the Lloyd and assign chunk calls)
//   XFORM   the whole (rows x k) block of distances / kernel values (bkm_transform_chunk)
//   COLSUM  per column j of the keep set: sum over rows of exp(-gamma d^2(x, c_j)) (bkm_kernel_colsum_chunk)
//   EMBED   per row: e = sum_j exp(-gamma (d^2(x, c_j) - min_j d^2)) W_j, written as e / ||e|| (bkm_nystrom_embed_chunk)
enum TcEpi { EPI_ARGMIN = 0, EPI_XFORM = 1, EPI_COLSUM = 2, EPI_EMBED = 3 };
static const int TC_EMBED_MAXK = 64;      // outputs of the EMBED epilogue (W rows are staged in shared memory)
// gamma * min_j d^2 beyond which the float64 reference's kernel row underflows to 0 everywhere (exp(-745.14) == 0 in
// float64): such rows are written as NaN, as the reference's 0 / 0 normalisation gives
static const double NYS_UNDERFLOW = 745.13;
// The Nystrom variants' configuration: per-warp column sums of a tile (COLSUM); the projection weights W [N][wp] fp32
// (EMBED: kw outputs, row pitch wp = ceil(kw/8)*8 + 4).  A type of its own, so that the ARGMIN / XFORM variants keep
// their parameter layout (and code) unchanged.
struct TcCfgNys : TcCfg {
  uint32_t off_cs, off_w;
  int kw, wp;
  const float* w;
};
template <int EPI> struct TcCfgOf { using type = TcCfg; };
template <> struct TcCfgOf<EPI_COLSUM> { using type = TcCfgNys; };
template <> struct TcCfgOf<EPI_EMBED> { using type = TcCfgNys; };

// The deferred-row re-check reports a failed fused kernel through this word (see tc_recheck_kernel); the wgmma kernel
// has no waits that can time out, so it stays 0 unless a debugging build sets it.
__device__ unsigned int g_tc_abort = 0;
__device__ unsigned int g_tc_dbg[64];

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int n) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// byte offset of X element (row r, feature f) in a ring slot
__device__ __forceinline__ uint32_t xsw(int r, int f) {
  return (uint32_t)((f >> 5) * XBOX_BYTES + r * 128 + ((((f >> 2) & 7) ^ (r & 7)) << 4) + (f & 3) * 4);
}
// M-step class-list entry of row `row` of a tile with label `c`: the byte offset of sums row c (bits 0-16) and the row's
// part of its slot offset, 128 row | (row & 7) << 4 (bits 17-31).  Rows of the sums are 64 floats, so a thread adds 8 f2
// (its feature pair 2 f2, 2 f2 + 1) to the first; to the second it applies the pair's swizzle, ^ ((f2 >> 1) & 7) << 4,
// and adds its box (f2 >> 4) and (f2 & 1) * 8.
static const int CLS_ROW_SHIFT = 17;
static const uint32_t CLS_SUM_MASK = (1u << CLS_ROW_SHIFT) - 1u;
static_assert((256 - 1) * 64 * 4 <= (int)CLS_SUM_MASK && ((TBM - 1) * 128 | 0x70) < (1 << (32 - CLS_ROW_SHIFT)), "class-list entry fields");
__device__ __forceinline__ uint32_t cls_entry(int c, int row) {
  return ((uint32_t)(row * 128 | (row & 7) << 4) << CLS_ROW_SHIFT) | (uint32_t)(c * 64 * 4);
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);          // low half = lower column
  return *reinterpret_cast<const uint32_t*>(&h);
}

// EPI (TcEpi): XFORM writes the whole (rows x k) block of distances / kernel values instead of the arg-min
// (euclidean_distances, dask_ml/metrics/pairwise.py:69-97; rbf_kernel :131-139); COLSUM and EMBED are the two passes
// of the Nystrom embedding (dask_ml/cluster/spectral.py:237-282).  Same MMAs, no M-step.
template <int N, int KS, bool MSTEP, bool WANT_DIST, int EPI>
__global__ void __launch_bounds__(128 * tc_warpgroups(MSTEP), 1)
tc_chunk_kernel(ChunkArgs a, typename TcCfgOf<EPI>::type cfg, const __grid_constant__ CUtensorMap xmap) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  extern __shared__ __align__(1024) unsigned char smem[];
  constexpr bool HAS_M = MSTEP || WANT_DIST;
  constexpr int NWG = tc_warpgroups(MSTEP), TC_THREADS = 128 * NWG;
  // N = 256: two MMA column halves of 128 (the second half's B rows start 128 x 128 bytes = 16 whole swizzle atoms on)
  constexpr int NH = N == 256 ? 2 : 1, NC = N / NH;
  const int tid = threadIdx.x, lane = tid & 31, wgi = tid >> 7, t = tid & 127, wq = t >> 5;
  const uint32_t sbase = smem_u32(smem);
  if (tid == 0 && (sbase & 1023)) __trap();                 // the swizzle pattern assumes 1024-byte aligned tiles
  const int d = a.d, k = a.k;
  float* cn_s = reinterpret_cast<float*>(smem + cfg.off_cn);          // [N] s^2 ||c||^2 (padded columns: 3e38)
  int* cnt_s = reinterpret_cast<int*>(smem + cfg.off_cnt);            // [N]
  float* sum_s = reinterpret_cast<float*>(smem + cfg.off_sum);        // [N][64]
  int* lab_s = reinterpret_cast<int*>(smem + cfg.off_lab) + wgi * TBM;        // label of each row of the tile, -1: none
  float* dp_s = reinterpret_cast<float*>(smem + cfg.off_dp) + wgi * 2 * TBM;  // [2][TBM] halves of the direct distances
  double* red_s = reinterpret_cast<double*>(smem + cfg.off_ring);    // teardown only: the ring is drained by then
  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const float sc = hdr->scale;
  const float inv_s = 1.0f / sc;                             // exact: s is a power of two, s and 1/s are normal
  const float gs = EPI != EPI_ARGMIN ? (float)(a.xf_gamma * (double)inv_s * (double)inv_s) : 0.f;   // rbf: gamma / s^2

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
    const float* cns = reinterpret_cast<const float*>(a.pack + a.L.off_cns);
    for (int j = tid; j < N; j += TC_THREADS) {
      cn_s[j] = j < a.L.kp ? cns[j] : 3.0e38f;
      cnt_s[j] = 0;
    }
    if (MSTEP)
      for (int i = tid; i < N * 64; i += TC_THREADS) sum_s[i] = 0.f;
    if constexpr (EPI == EPI_EMBED) {
      // W rows j < k (keep rows), outputs o < kw; zero elsewhere
      float* w_s = reinterpret_cast<float*>(smem + cfg.off_w);
      for (int i = tid; i < N * cfg.wp; i += TC_THREADS) {
        const int j = i / cfg.wp, o = i - j * cfg.wp;
        w_s[i] = (j < k && o < cfg.kw) ? cfg.w[(size_t)j * cfg.kw + o] : 0.f;
      }
    }
    wg::fence_proxy_async();                                 // generic-proxy stores -> visible to wgmma
  }
  const long long ntiles = (a.n + TBM - 1) / TBM;
  const long long my_tiles = blockIdx.x < ntiles ? (ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
  const long long nrounds = (my_tiles + NWG - 1) / NWG;      // warpgroup w takes the CTA's tiles NWG p + w
  const int S = cfg.S;
  const uint32_t bar0 = sbase + cfg.off_bar, ring0 = sbase + cfg.off_ring;
  // tile lt -> slot lt % S: its ceil(d / 32) boxes, completion counted in bytes on the slot's mbarrier
  auto load_tile = [&](long long lt, int slot) {
    const uint32_t bar = bar0 + 8u * (uint32_t)slot, dst = ring0 + (uint32_t)slot * XSLOT_BYTES;
    const int row0 = (int)((blockIdx.x + lt * gridDim.x) * TBM);
    constexpr int nbox = (KS + 1) / 2;
    ptx::mbar_expect_tx(bar, nbox * XBOX_BYTES);
#pragma unroll
    for (int b = 0; b < nbox; ++b) ptx::tma_load_2d(dst + b * XBOX_BYTES, &xmap, 32 * b, row0, bar);
  };
  if (tid == 0) {
    for (int i = 0; i < S; ++i) ptx::mbar_init(bar0 + 8u * i, 1);
    ptx::mbar_fence_init();
    for (int lt = 0; lt < S && lt < my_tiles; ++lt) load_tile(lt, lt);
  }
  __syncthreads();

  const int g = lane >> 2, c2 = (lane & 3) * 2;
  const int rA = wq * 16 + g;                                // this thread's accumulator rows: rA, rA + 8
  const uint64_t dbh = wg::desc_sw128(sbase + cfg.off_bhi), dbl = wg::desc_sw128(sbase + cfg.off_blo);
  const float cnmax = (float)(hdr->cn_max * (double)sc * (double)sc);
  double dsum = 0.0;
  double cs0 = 0.0, cs1 = 0.0;                               // COLSUM: this warpgroup's sums of columns t, t + 128

  int slot = wgi;                                            // lt % S and the parity (lt / S) & 1 of the slot's fill
  uint32_t fill = 0;
#pragma unroll 1
  for (long long p = 0; p < nrounds; ++p) {
    const long long lt = NWG * p + wgi;
    const bool has = lt < my_tiles;
    const long long row0 = (blockIdx.x + lt * gridDim.x) * TBM;
    unsigned char* xs = smem + cfg.off_ring + (uint32_t)slot * XSLOT_BYTES;
    // The previous fill of this slot (tile lt - S) must have landed before this wait starts: if it has not, the
    // barrier is still in that phase, and the parity of tile lt's phase, which is also that of tile lt - 2S's, reads as
    // complete.  Without the M-step (two warpgroups, S even, see place_ring) tile lt - S is this warpgroup's own
    // earlier tile.  With it (three warpgroups, any S >= 4) the turn order covers it: this warpgroup's previous turn
    // (tile lt - 3) came after the turns of tiles lt - 4, lt - 5, ..., lt - S, and the turn of tile lt - S came after
    // its warpgroup's wait for that tile.
    if (has) ptx::mbar_wait(bar0 + 8u * (uint32_t)slot, fill);
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
            const float2 v = *reinterpret_cast<const float2*>(xs + xsw(rA + (h & 1) * 8, s * 16 + c2 + (h >> 1) * 8));
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

      // ---- acc = Xhi.Bhi + Xhi.Blo + Xlo.Bhi of columns [hf NC, (hf + 1) NC) into ah, one commit group ----
      auto mma_half = [&](float(&ah)[NC / 2], int hf) {
        const uint64_t bh = dbh + (uint64_t)(hf * NC * 128 / 16), bl = dbl + (uint64_t)(hf * NC * 128 / 16);
#pragma unroll
        for (int s = 0; s < KS; ++s) wg::Mma<NC>::rs_f16(ah, ahi[s], bh + (uint64_t)(2 * s), s > 0);
#pragma unroll
        for (int s = 0; s < KS; ++s) wg::Mma<NC>::rs_f16(ah, ahi[s], bl + (uint64_t)(2 * s), 1);
#pragma unroll
        for (int s = 0; s < KS; ++s) wg::Mma<NC>::rs_f16(ah, alo[s], bh + (uint64_t)(2 * s), 1);
        wg::commit();
      };
      // the whole tile's accumulators (the epilogues other than the arg-min): the accumulator fragment of columns
      // [hf NC, (hf + 1) NC) is acc[hf NC / 2 ...]
      constexpr int NACC = EPI == EPI_ARGMIN ? NC : N;
      float acc[NACC / 2];
#pragma unroll
      for (int i = 0; i < NACC / 2; ++i) acc[i] = 0.f;
      if constexpr (EPI != EPI_ARGMIN) {
        wg::fence();
#pragma unroll
        for (int hf = 0; hf < NH; ++hf) mma_half(*reinterpret_cast<float(*)[NC / 2]>(acc + hf * (NC / 2)), hf);
      }

      if constexpr (EPI == EPI_COLSUM) {
        wg::wait_all();
        wg::pin(acc);
        // v = exp(-(gamma / s^2) y) of the tile's real rows; per column the warp's 16 rows are added by a fixed shuffle
        // tree (rows rA, rA + 8 in the thread, then lanes g = 0..7), the 4 warps' sums in warp order, all in fp32; the
        // tile's sum then goes into the thread's float64 accumulator of that column
        const bool ok0 = row0 + rA < a.n, ok1 = row0 + rA + 8 < a.n;
        float* cs_s = reinterpret_cast<float*>(smem + cfg.off_cs) + wgi * 4 * N;     // [4 warps][N]
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * i + c2 + e;
            float v = ok0 ? __expf(-gs * fmaxf((acc[4 * i + e] + cn_s[col]) + xn0, 0.f)) : 0.f;
            if (ok1) v += __expf(-gs * fmaxf((acc[4 * i + 2 + e] + cn_s[col]) + xn1, 0.f));
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);
            v += __shfl_xor_sync(0xffffffffu, v, 16);
            if (g == 0) cs_s[wq * N + col] = v;
          }
        }
        wg::wg_sync(1 + wgi);
        if (t < N) cs0 += (double)(((cs_s[t] + cs_s[N + t]) + cs_s[2 * N + t]) + cs_s[3 * N + t]);
        if (t + 128 < N) cs1 += (double)(((cs_s[t + 128] + cs_s[N + t + 128]) + cs_s[2 * N + t + 128]) + cs_s[3 * N + t + 128]);
      } else if constexpr (EPI == EPI_EMBED) {
        wg::wait_all();
        wg::pin(acc);
        // y (clamped at 0) and the row minimum m over the real columns (the quad holds a row's columns)
        float m0 = CUDART_INF_F, m1 = CUDART_INF_F;
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * i + c2 + e;
            const float y0 = fmaxf((acc[4 * i + e] + cn_s[col]) + xn0, 0.f);
            const float y1 = fmaxf((acc[4 * i + 2 + e] + cn_s[col]) + xn1, 0.f);
            acc[4 * i + e] = y0; acc[4 * i + 2 + e] = y1;
            if (col < k) { m0 = fminf(m0, y0); m1 = fminf(m1, y1); }
          }
        }
        m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fminf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
        m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fminf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
        // v = exp(-(gamma / s^2)(y - m)): the largest term of a row is 1, so fp32 does not underflow where the float64
        // reference does not (the shift cancels in the normalisation)
#pragma unroll
        for (int i = 0; i < N / 8; ++i) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const bool real = 8 * i + c2 + e < k;
            acc[4 * i + e] = real ? __expf(-gs * (acc[4 * i + e] - m0)) : 0.f;
            acc[4 * i + 2 + e] = real ? __expf(-gs * (acc[4 * i + 2 + e] - m1)) : 0.f;
          }
        }
        // e = v . W in groups of 8 outputs: per thread over its columns, then the quad's 4 partial sums (the same
        // value lands in all 4 lanes); lane q of the quad stages outputs 2q, 2q + 1 of the group in the tile's X
        // slot (rows of this warp only: their A fragments are built and consumed)
        const float* w_s = reinterpret_cast<const float*>(smem + cfg.off_w);
        const int q = lane & 3;
        float n0 = 0.f, n1 = 0.f;
        __syncwarp();
#pragma unroll 1
        for (int o0 = 0; o0 < cfg.kw; o0 += 8) {
          float e0[8], e1[8];
#pragma unroll
          for (int o = 0; o < 8; ++o) { e0[o] = 0.f; e1[o] = 0.f; }
#pragma unroll
          for (int i = 0; i < N / 8; ++i) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const float* wr = w_s + (8 * i + c2 + e) * cfg.wp + o0;
              const float4 wa = *reinterpret_cast<const float4*>(wr), wb = *reinterpret_cast<const float4*>(wr + 4);
              const float w8[8] = {wa.x, wa.y, wa.z, wa.w, wb.x, wb.y, wb.z, wb.w};
              const float va = acc[4 * i + e], vb = acc[4 * i + 2 + e];
#pragma unroll
              for (int o = 0; o < 8; ++o) { e0[o] = fmaf(va, w8[o], e0[o]); e1[o] = fmaf(vb, w8[o], e1[o]); }
            }
          }
#pragma unroll
          for (int o = 0; o < 8; ++o) {
            e0[o] += __shfl_xor_sync(0xffffffffu, e0[o], 1); e0[o] += __shfl_xor_sync(0xffffffffu, e0[o], 2);
            e1[o] += __shfl_xor_sync(0xffffffffu, e1[o], 1); e1[o] += __shfl_xor_sync(0xffffffffu, e1[o], 2);
            n0 = fmaf(e0[o], e0[o], n0); n1 = fmaf(e1[o], e1[o], n1);       // outputs >= kw are 0 (W is zero padded)
          }
          const float2 p0 = q == 0 ? make_float2(e0[0], e0[1]) : q == 1 ? make_float2(e0[2], e0[3])
                          : q == 2 ? make_float2(e0[4], e0[5]) : make_float2(e0[6], e0[7]);
          const float2 p1 = q == 0 ? make_float2(e1[0], e1[1]) : q == 1 ? make_float2(e1[2], e1[3])
                          : q == 2 ? make_float2(e1[4], e1[5]) : make_float2(e1[6], e1[7]);
          *reinterpret_cast<float2*>(xs + xsw(rA, o0 + 2 * q)) = p0;
          *reinterpret_cast<float2*>(xs + xsw(rA + 8, o0 + 2 * q)) = p1;
        }
        // per-row factor 1 / ||e||; NaN where gamma * m (unscaled, float64) is beyond the float64 reference's underflow
        if (q == 0) {
          const double gsd = a.xf_gamma * (double)inv_s * (double)inv_s;
          dp_s[rA] = ((double)m0 * gsd > NYS_UNDERFLOW) ? CUDART_NAN_F : 1.0f / sqrtf(n0);
          dp_s[rA + 8] = ((double)m1 * gsd > NYS_UNDERFLOW) ? CUDART_NAN_F : 1.0f / sqrtf(n1);
        }
        __syncwarp();
        // the warp writes its 16 rows, consecutive lanes on consecutive outputs
        const int kw = cfg.kw;
        for (int e = lane; e < 16 * kw; e += 32) {
          const int rr = e / kw, o = e - rr * kw, r = wq * 16 + rr;
          const long long row = row0 + r;
          if (row < a.n) __stcs(a.xf_out + row * a.xf_ld + o, *reinterpret_cast<const float*>(xs + xsw(r, o)) * dp_s[r]);
        }
        ptx::fence_proxy_async();                            // these generic writes before the slot's next TMA fill
      } else if constexpr (EPI == EPI_XFORM) {
        wg::wait_all();
        wg::pin(acc);
        // y = acc + s^2 ||c||^2 + ||s x||^2 = s^2 d^2, clamped at 0; mode 0: sqrt(y) / s, 1: y / s / s, 2: exp(-(gamma /
        // s^2) y).  1/s is a normal float (pack_scale_exp) but 1/s^2 need not be, so it is never formed in fp32.
        // One copy of the store loop per mode, so that each element pays for its own mode's arithmetic only
        const bool vec_ok = ((reinterpret_cast<uintptr_t>(a.xf_out) & 7) == 0) && ((a.xf_ld & 1) == 0);
        auto store_block = [&](auto value) {
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
              for (int e = 0; e < 2; ++e) o[e] = value(fmaxf((acc[4 * i + 2 * h + e] + cn_s[col + e]) + xn, 0.f));
              if (vec_ok && col + 1 < k) __stcs(reinterpret_cast<float2*>(orow + col), make_float2(o[0], o[1]));
              else {
                if (col < k) orow[col] = o[0];
                if (col + 1 < k) orow[col + 1] = o[1];
              }
            }
          }
        };
        if (a.xf_mode == 0) store_block([&](float y) { return sqrtf(y) * inv_s; });
        else if (a.xf_mode == 1) store_block([&](float y) { return (y * inv_s) * inv_s; });
        else store_block([&](float y) { return __expf(-gs * y); });
      } else {
        static_assert(EPI == EPI_ARGMIN, "epilogue");
        // ---- arg-min, near-tie test (bound = tau (||s x||^2 + max ||s c||^2)), one column half at a time: the row
        //      minimum m of the half, then the count and index sum of its columns with value <= thr = m + bound over
        //      the columns so far (tau >= 0; xn >= 0 or NaN) ----
        float m[2] = {CUDART_INF_F, CUDART_INF_F}, thr[2], hits[2] = {0.f, 0.f};
        const float xb[2] = {xn0 + cnmax, xn1 + cnmax};
#pragma unroll
        for (int hf = 0; hf < NH; ++hf) {
          wg::fence();                                       // the registers of the previous half were written
          mma_half(acc, hf);
          wg::wait_all();
          wg::pin(acc);
          wg::near_tie_cols<NC>(acc, cn_s, hf * NC, lane, a.tau, xb, m, thr, hits);
        }
        wg::hit_quad_merge(hits, lane);
        if ((lane & 3) == 0) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float xn = h ? xn1 : xn0;
            const int r = rA + 8 * h;
            const long long row = row0 + r;
            // an entry beyond fp16's range (|s x| >= 65504 => xn >= 4.29e9) or a non-finite one: float64 path
            const bool out_of_range = !(xn < 4.29e9f);
            // a near-tie iff the second best is <= thr, i.e. iff not exactly one column is <= thr; a thr that is +inf
            // or NaN makes every row a near-tie, as the comparison with the second best does
            const bool tie = !(hits[h] >= 1.f && hits[h] < 2.f) || !(thr[h] < CUDART_INF_F) || out_of_range;
            const int j = (int)((hits[h] - 1.f) * 1024.f);  // the arg-min when exactly one column is <= thr
            const bool valid = row < a.n;
            const bool flagged = valid && tie && k > 1;
            const int bj = (tie || j >= k) ? 0 : j;
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
        // winning distance in direct form sum (s x - s c)^2 (fp32 centres of the pack): thread (row r, feature half
        // hh), features visited in a per-row rotated order so that the 32 rows of a warp hit 32 different banks.  It is
        // formed in the scaled domain, where a row that was not deferred has every |s x| < 2^16: it cannot overflow, and
        // it does not depend on the magnitude of the data (the scale follows the centres).  The square root is taken
        // there too, and 1/s (1/s^2) is applied in float64, so no intermediate leaves the float range
        const int r = t & 63, hh = t >> 6;
        const int lab = lab_s[r];
        float s0 = 0.f, s1 = 0.f;
        if (lab >= 0) {
          const float* cr = reinterpret_cast<const float*>(a.pack + a.L.off_cT) + (size_t)lab * a.L.d4;
#pragma unroll 8
          for (int i = 0; i < 32; i += 2) {
            const int f0 = hh * 32 + ((i + r) & 31), f1 = hh * 32 + ((i + 1 + r) & 31);
            if (f0 < d) { const float e = fmaf(sc, *reinterpret_cast<const float*>(xs + xsw(r, f0)), -(sc * cr[f0])); s0 = fmaf(e, e, s0); }
            if (f1 < d) { const float e = fmaf(sc, *reinterpret_cast<const float*>(xs + xsw(r, f1)), -(sc * cr[f1])); s1 = fmaf(e, e, s1); }
          }
        }
        dp_s[hh * TBM + r] = s0 + s1;
        wg::wg_sync(1 + wgi);
        if (t < TBM && lab >= 0) {
          const float y = dp_s[t] + dp_s[TBM + t];                            // s^2 d^2
          const double outv = a.squared ? (double)y * (double)inv_s * (double)inv_s : (double)sqrtf(y) * (double)inv_s;
          dsum += outv;
          if (a.min_out) reinterpret_cast<float*>(a.min_out)[row0 + t] = (float)outv;
        }
      }
      if (MSTEP) {
        // thread (feature pair f2, class q) owns sums[c][2 f2] and sums[c][2 f2 + 1] of the clusters c with c % 4 == q,
        // where q is the warp's index in its warpgroup: a warp covers all 64 features of one class, in 64-bit accesses.
        // Before its turn each warp lists the tile's rows of its class in row order, as byte offsets (cls_entry);
        // deferred rows are left out.  Then it marks the list positions whose label repeats an earlier one of the same
        // batch of 8
        const int f2 = lane, q = wq;
        uint32_t* cls = reinterpret_cast<uint32_t*>(smem + cfg.off_cls) + (tid >> 5) * TBM;
        int ncls = 0;
        uint64_t rep = 0;                                    // bit i: list position i repeats a label of its batch
        if (has) {
          const int la = lab_s[lane], lb = lab_s[32 + lane];
          const unsigned ma = __ballot_sync(0xffffffffu, la >= 0 && (la & 3) == q);
          const unsigned mb = __ballot_sync(0xffffffffu, lb >= 0 && (lb & 3) == q);
          const unsigned lt = (1u << lane) - 1u;
          if ((ma >> lane) & 1u) cls[__popc(ma & lt)] = cls_entry(la, lane);
          if ((mb >> lane) & 1u) cls[__popc(ma) + __popc(mb & lt)] = cls_entry(lb, 32 + lane);
          ncls = __popc(ma) + __popc(mb);
          __syncwarp();
          for (int h = 0; h < 2 && 32 * h < ncls; ++h) {
            const int pos = 32 * h + lane;
            const uint32_t c = cls[pos] & CLS_SUM_MASK;
            bool r = false;
#pragma unroll
            for (int s = 1; s < 8; ++s) {
              const uint32_t o = __shfl_up_sync(0xffffffffu, c, s);   // position pos - s
              r |= (lane & 7) >= s && o == c;
            }
            rep |= (uint64_t)__ballot_sync(0xffffffffu, r && pos < ncls) << (32 * h);
          }
        }
        // turn order of the CTA's M-steps: the tile order lt = 0, 1, 2, ... (warpgroup 0 round p, warpgroup 1 round p,
        // ..., warpgroup 0 round p + 1, ...; a round past the CTA's last tile takes its turn with an empty list).  Only
        // warp w of the other warpgroups owns the same sums elements, so the order is kept per warp triple: named
        // barrier 1 + NWG + NWG w + i hands warp w's turn from warpgroup i to warpgroup i + 1 mod NWG (ids 4 .. 15;
        // 1 .. 3 are the warpgroups' own).  A barrier is not reused before its previous use completes: warpgroup i
        // arrives at it again only after its own next turn, which waited on the whole cycle.
        static_assert(1 + NWG + NWG * 4 <= 16, "named barriers");
        if (lt > 0) bar_sync(1 + NWG + NWG * wq + (wgi + NWG - 1) % NWG, 64);
        // the rows of the list go in 8 at a time: the batch's sums are read before any is written; in a batch with a
        // repeated label, a row continues from the running sum of that label's earlier row.  So every element receives
        // its rows in tile order, then row order, one rounded addition each.  The positions of the last batch beyond
        // the list are not accessed (the list is not padded: a padding row would cost shared-memory traffic like a
        // real one).  A pair that straddles d also adds the zero-filled column d into its second element, which the
        // teardown never reads
        if (2 * f2 < d) {
          const uint32_t fo = (uint32_t)f2 * 8u, fx = (uint32_t)((f2 >> 1) & 7) << 4;
          unsigned char* sum_b = reinterpret_cast<unsigned char*>(sum_s);
          const unsigned char* xs_b = xs + (f2 >> 4) * XBOX_BYTES + (f2 & 1) * 8;
          const uint4* cl4 = reinterpret_cast<const uint4*>(cls);
          uint4 ea = cl4[0], eb = cl4[1];
#pragma unroll 1
          for (int b = 0; 8 * b < ncls; ++b) {
            const uint32_t e[8] = {ea.x, ea.y, ea.z, ea.w, eb.x, eb.y, eb.z, eb.w};
            const int nb = ncls - 8 * b;                     // list rows in this batch (warp-uniform)
            float2 v[8], x[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              v[j] = x[j] = make_float2(0.f, 0.f);
              if (j < nb) {
                v[j] = *reinterpret_cast<const float2*>(sum_b + ((e[j] & CLS_SUM_MASK) | fo));
                x[j] = *reinterpret_cast<const float2*>(xs_b + ((e[j] >> CLS_ROW_SHIFT) ^ fx));
              }
            }
            if (8 * (b + 1) < ncls) { ea = cl4[2 * b + 2]; eb = cl4[2 * b + 3]; }
            if ((rep >> (8 * b)) & 0xffu) {
#pragma unroll
              for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int i = 0; i < j; ++i)
                  if (((e[i] ^ e[j]) & CLS_SUM_MASK) == 0u) v[j] = v[i];
                v[j].x += x[j].x; v[j].y += x[j].y;
              }
            } else {
#pragma unroll
              for (int j = 0; j < 8; ++j) { v[j].x += x[j].x; v[j].y += x[j].y; }
            }
            // a repeated label: the last store is the full sum
#pragma unroll
            for (int j = 0; j < 8; ++j)
              if (j < nb) *reinterpret_cast<float2*>(sum_b + ((e[j] & CLS_SUM_MASK) | fo)) = v[j];
          }
        }
        // bar.arrive -> bar.sync orders these shared-memory writes before the next turn's accesses (PTX memory model:
        // the arrive synchronizes with the sync on the same barrier)
        if (lt + 1 < NWG * nrounds) bar_arrive(1 + NWG + NWG * wq + wgi, 64);
      }
    }
    wg::wg_sync(1 + wgi);                                    // the slot and lab_s may be refilled
    if (t == 0 && lt + S < my_tiles) {
      ptx::fence_proxy_async();                              // the warpgroup's accesses to the slot before the async-proxy fill
      load_tile(lt + S, slot);
    }
    slot += NWG;                                             // NWG < S: at most one wrap
    if (slot >= S) { slot -= S; fill ^= 1u; }
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
  if constexpr (EPI == EPI_COLSUM) {
    // partial column sums of warpgroup wgi of this CTA -> slot 2 * CTA + wgi (colsum_fold adds the slots in order)
    double* part = a.pin + (size_t)(2 * blockIdx.x + wgi) * k;
    if (t < k) part[t] = cs0;
    if (t + 128 < k) part[t + 128] = cs1;
    return;
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
  // any d <= 64: columns beyond d are zero-filled when a tile is staged; what the TMA copies do need is a
  // 16-byte row pitch and base (launch_tc returns BKM_EALIGN otherwise and the caller falls back to the CUDA-core
  // kernel), which the host side provides by uploading row chunks with a padded pitch (engine.CudaBackend.to_device)
  return dtype == BKM_F32 && d >= 1 && d <= 64 && k >= 1 && k <= 256;
}

// The arrays of every variant; returns the end of the last one
static uint32_t layout_common(int d, int k, bool mstep, TcCfg* c) {
  c->KS = (d + 15) / 16;
  c->NP = (k + 15) / 16 * 16;
  const uint32_t N = (uint32_t)wg::mma_n(c->NP);
  uint32_t o = 0;
  c->off_bhi = o; o += N * 128u;                    // fp16 B tiles: N rows x 64 halves (one 128-byte swizzle atom)
  c->off_blo = o; o += N * 128u;
  c->off_sum = o; if (mstep) o += N * 64u * 4u;          // per-CTA sums [N][64]
  c->off_cn = o; o += N * 4u;
  c->off_cnt = o; o += N * 4u;
  const uint32_t nwg = (uint32_t)tc_warpgroups(mstep);
  c->off_lab = o; o += nwg * TBM * 4u;              // per warpgroup: the labels of its tile
  c->off_dp = o; o += nwg * 2u * TBM * 4u;          // per warpgroup: halves of the direct distances
  c->off_cls = o; if (mstep) o += nwg * 4u * TBM * 4u;   // per-warp class lists of the M-step
  return o;
}
// The X ring fills what is left of the 227 KB from offset o: S = as many 16 KB slots as fit (at most TC_MAX_STAGES).
// Without the M-step turns nothing orders the two warpgroups, so S is rounded down to even there: each slot is then
// filled and read by one warpgroup only.  The M-step variants' three warpgroups are ordered by their turns, which
// covers any S >= 4 (see the wait in tc_chunk_kernel)
static bool place_ring(TcCfg* c, uint32_t o, bool mstep) {
  const uint32_t cap = 227u * 1024u;
  c->off_bar = o; o += TC_MAX_STAGES * 8u;           // one "full" mbarrier per slot
  o = (o + 1023u) & ~1023u;                          // the swizzle pattern repeats every 1024 bytes
  c->off_ring = o;
  c->S = o < cap ? (int)min((uint32_t)TC_MAX_STAGES, (cap - o) / XSLOT_BYTES) : 0;
  if (!mstep) c->S &= ~1;
  c->total = o + (uint32_t)c->S * XSLOT_BYTES;
  static_assert(TC_MAX_THREADS * 8u <= XSLOT_BYTES, "the teardown's reduction array lives in the first slot");
  return c->S >= TC_MIN_STAGES;
}

static bool make_cfg(int d, int k, bool mstep, TcCfg* c) { return place_ring(c, layout_common(d, k, mstep, c), mstep); }

static bool make_cfg_nys(int d, int k, int epi, int kw, TcCfgNys* c) {
  const uint32_t N = (uint32_t)wg::mma_n((k + 15) / 16 * 16);
  uint32_t o = layout_common(d, k, false, c);
  c->off_cs = o; if (epi == EPI_COLSUM) o += 2u * 4u * N * 4u;     // per-warp column sums of a tile
  c->kw = kw;
  c->wp = (kw + 7) / 8 * 8 + 4;                     // 4 mod 8 floats: the quad's 4 W rows of a float4 load hit 4 bank groups
  c->w = nullptr;
  c->off_w = o; if (epi == EPI_EMBED) o += N * (uint32_t)c->wp * 4u;   // (every offset above is a multiple of 16)
  return place_ring(c, o, false);
}

// Tensor map of the chunk for the ring's TMA fills: fp32 (d, n) with row pitch ldx, boxes of 32 columns x 64 rows,
// SWIZZLE_128B; the copy engine zero-fills what lies beyond d or n.  The encoder is the driver's, reached through the
// runtime (the library links cudart statically and no driver library).
static int encode_x_map(const ChunkArgs& a, CUtensorMap* m) {
  static PFN_cuTensorMapEncodeTiled_v12000 encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    BKM_CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    if (q != cudaDriverEntryPointSuccess || !fn) return BKM_EUNSUPPORTED;
    encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
  const cuuint64_t dims[2] = {(cuuint64_t)a.d, (cuuint64_t)(a.n > 0 ? a.n : 1)};
  const cuuint64_t strides[1] = {(cuuint64_t)a.ldx * 4u};
  const cuuint32_t box[2] = {32u, (cuuint32_t)TBM}, estr[2] = {1u, 1u};
  const CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(a.X), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : BKM_EUNSUPPORTED;
}

template <int N, int KS, bool M, bool W, int XF>
static int launch_variant(const ChunkArgs& a, const typename TcCfgOf<XF>::type& cfg, int grid, cudaStream_t s) {
  CUtensorMap xmap;
  if (const int rc = encode_x_map(a, &xmap)) return rc;
  auto kern = tc_chunk_kernel<N, KS, M, W, XF>;
  BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.total));
  kern<<<grid, 128 * tc_warpgroups(M), cfg.total, s>>>(a, cfg, xmap);
  return 0;
}
template <int N, bool M, bool W, int XF>
static int launch_ks(const ChunkArgs& a, const typename TcCfgOf<XF>::type& cfg, int grid, cudaStream_t s) {
  switch (cfg.KS) {
    case 1: return launch_variant<N, 1, M, W, XF>(a, cfg, grid, s);
    case 2: return launch_variant<N, 2, M, W, XF>(a, cfg, grid, s);
    case 3: return launch_variant<N, 3, M, W, XF>(a, cfg, grid, s);
    default: return launch_variant<N, 4, M, W, XF>(a, cfg, grid, s);
  }
}
template <bool M, bool W, int XF>
static int launch_n(const ChunkArgs& a, const typename TcCfgOf<XF>::type& cfg, int grid, cudaStream_t s) {
  switch (wg::mma_n(cfg.NP)) {
    case 16: return launch_ks<16, M, W, XF>(a, cfg, grid, s);
    case 32: return launch_ks<32, M, W, XF>(a, cfg, grid, s);
    case 64: return launch_ks<64, M, W, XF>(a, cfg, grid, s);
    case 128: return launch_ks<128, M, W, XF>(a, cfg, grid, s);
    default: return launch_ks<256, M, W, XF>(a, cfg, grid, s);
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
  if (mstep) rc = want_dist ? launch_n<true, true, EPI_ARGMIN>(a, cfg, grid, s) : launch_n<true, false, EPI_ARGMIN>(a, cfg, grid, s);
  else rc = want_dist ? launch_n<false, true, EPI_ARGMIN>(a, cfg, grid, s) : launch_n<false, false, EPI_ARGMIN>(a, cfg, grid, s);
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
  const int rc = launch_n<false, false, EPI_XFORM>(a, cfg, tc_grid(a.n, sm_count), s);
  if (rc) return rc;
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// Nystrom column sums on the tensor path: per-warpgroup partials [2 * grid][k] (float64) into `part`; returns the number
// of partial slots written, which colsum_fold adds in slot order
int launch_tc_colsum(const ChunkArgs& a, double* part, size_t part_bytes, int sm_count, int* parts_out, cudaStream_t s) {
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || (a.ldx % 4)) return BKM_EALIGN;
  TcCfgNys cfg;
  if (!make_cfg_nys(a.d, a.k, EPI_COLSUM, 0, &cfg)) return BKM_EUNSUPPORTED;
  const int grid = tc_grid(a.n, sm_count);
  if ((size_t)2 * grid * a.k * sizeof(double) > part_bytes) return BKM_EWORKSPACE;
  ChunkArgs b = a;
  b.pin = part;
  const int rc = launch_n<false, false, EPI_COLSUM>(b, cfg, grid, s);
  if (rc) return rc;
  *parts_out = 2 * grid;
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

// Nystrom embedding rows on the tensor path (kw <= TC_EMBED_MAXK outputs, W fp32 [k][kw]); out = a.xf_out, pitch a.xf_ld
int launch_tc_embed(const ChunkArgs& a, const float* W, int kw, int sm_count, cudaStream_t s) {
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || (a.ldx % 4)) return BKM_EALIGN;
  if (kw < 1 || kw > TC_EMBED_MAXK) return BKM_EUNSUPPORTED;
  TcCfgNys cfg;
  if (!make_cfg_nys(a.d, a.k, EPI_EMBED, kw, &cfg)) return BKM_EUNSUPPORTED;
  cfg.w = W;
  const int rc = launch_n<false, false, EPI_EMBED>(a, cfg, tc_grid(a.n, sm_count), s);
  if (rc) return rc;
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace bkm

// The variant of tc_chunk_kernel a call would run, from the same configuration functions the launches use
extern "C" int bkm_debug_tc_layout(int d, int k, int epi, int mstep, int kw, int* out4) {
  using namespace bkm;
  if (!out4 || epi < EPI_ARGMIN || epi > EPI_EMBED || (mstep && epi != EPI_ARGMIN)) return BKM_EINVAL;
  if (!tc_supported(d, k, BKM_F32)) return BKM_EUNSUPPORTED;
  TcCfgNys c;
  bool ok;
  if (epi == EPI_ARGMIN || epi == EPI_XFORM) ok = make_cfg(d, k, mstep != 0, &c);
  else if (epi == EPI_COLSUM) ok = make_cfg_nys(d, k, EPI_COLSUM, 0, &c);
  else ok = kw >= 1 && kw <= TC_EMBED_MAXK && make_cfg_nys(d, k, EPI_EMBED, kw, &c);
  if (!ok) return BKM_EUNSUPPORTED;
  out4[0] = c.KS;
  out4[1] = wg::mma_n(c.NP);
  out4[2] = c.S;
  out4[3] = (int)c.total;
  return 0;
}

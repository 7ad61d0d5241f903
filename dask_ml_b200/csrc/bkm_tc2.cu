// bkm_tc2.cu — E-step on the Hopper tensor cores (wgmma, sm_90a) for LARGE shapes: bf16 rows, any k, d <= 128
// (BASELINE config C5: bf16 rows, d = 128, k = 1024 — the tensor-bound configuration).
//
// Reference operator: sklearn pairwise_distances_argmin_min(x, centers) per chunk (dask_ml/metrics/pairwise.py:35-38).
//
// Layout of the work ("B-stationary"): the k centres are cut into S = ceil(k / 256) slices of NS <= 256 centres.
// CTA b serves slice b % S for the row tiles of group b / S (G = SMs / S groups): its slice of -2 C, as a bf16
// (hi, lo) pair per 64-feature K-block, is loaded ONCE and stays resident in shared memory (128 KB at NS = 256,
// d = 128); the kernel then streams 64-row bf16 tiles of X (cp.async, double-buffered per warpgroup) and computes, per
// tile,
//     acc[64 x NS] = X . (-2 C)_hi^T  +  X . (-2 C)_lo^T          (fp32 accumulators in registers)
// plus ||c||^2 per column in the epilogue.  X is multiplied as it lies in HBM (bf16 operands, no scaling: bf16 has
// fp32's range); the centres carry 16 significant bits through the bf16 pair (representation error <= 2^-18 |c|),
// which the near-tie bound accounts for (tau_for, bkm_api.cu).  wgmma needs A and B in the same 16-bit format, so the
// centre splits are bf16 like the rows.  Each centre slice is read from L2 once per CTA, X tiles are read by the S
// CTAs of a group at about the same time (one HBM read, S - 1 L2 hits).
//
// CTA = 2 warpgroups, 1 CTA per SM; each warpgroup owns alternate tiles: row norms ||x||^2 from the staged tile,
// 2 ceil(d/16) wgmma.m64nNk16 (A and B from SWIZZLE_128B shared memory), the arg-min epilogue from registers.
// S == 1: the epilogue decides the row (label, or deferred to the float64 re-check).  S > 1: it writes a partial
// record {m1, label-or-tie, ||x||^2} per (slice, row); tc2_combine_kernel folds the S records of a row.
// The M-step and the winning distances for these shapes are label-indexed row passes (bkm_rowpass.cu): k * d partial
// sums (512 KB at C5) do not fit a CTA, so the sums are accumulated by cluster slice in a second sweep.
#include "bkm_common.cuh"
#include "bkm_wgmma.cuh"
#include <cuda_bf16.h>
#include <math_constants.h>

namespace bkm {

static const int T2_BM = 64;          // rows per warpgroup tile (wgmma M)
static const int T2_THREADS = 256;    // two warpgroups

struct Tc2Cfg {
  int S, NS, KB, KS;        // slices, slice width, 64-element K-blocks, 16-element K-steps (ceil(d/16))
  int G;                    // row-tile groups (grid = G * S)
  uint32_t off_b, off_x, off_cn, off_xn, total;
};

template <int N>
__global__ void __launch_bounds__(T2_THREADS, 1)
tc2_assign_kernel(ChunkArgs a, Tc2Cfg cfg) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, wgi = tid >> 7, t = tid & 127, wq = t >> 5;
  const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(smem);
  if (tid == 0 && (sbase & 1023)) __trap();                 // the swizzle pattern assumes 1024-byte aligned tiles
  const int S = cfg.S, NS = cfg.NS, KB = cfg.KB, d = a.d;
  const int slice = blockIdx.x % S, group = blockIdx.x / S;
  const uint32_t btile = (uint32_t)N * 128u;                // one (variant, K-block) tile of the slice
  const uint32_t xkblk = T2_BM * 128u;                      // one K-block of a staged X tile
  const uint32_t stage_bytes = (uint32_t)KB * xkblk;
  float* cn_s = reinterpret_cast<float*>(smem + cfg.off_cn);            // [N] ||c||^2 of the slice (padded: 3e38)
  float* xn_s = reinterpret_cast<float*>(smem + cfg.off_xn) + wgi * 2 * T2_BM;   // [2][T2_BM] halves of ||x||^2

  // ---------------- setup: the slice's B tiles and ||c||^2 ----------------
  {
    const int rq = KB * 8;                                  // 16-byte chunks per pack row ([kp2][KB * 64] bf16)
    const uint4* ghi = reinterpret_cast<const uint4*>(a.pack + a.L.off_b2hi);
    const uint4* glo = reinterpret_cast<const uint4*>(a.pack + a.L.off_b2lo);
    for (int i = tid; i < 2 * KB * N * 8; i += T2_THREADS) {
      const int v = i / (KB * N * 8), rem = i - v * (KB * N * 8);
      const int kb = rem / (N * 8), r = (rem - kb * N * 8) >> 3, q = rem & 7;
      uint4 val = make_uint4(0u, 0u, 0u, 0u);
      if (r < NS) val = (v ? glo : ghi)[(size_t)(slice * NS + r) * rq + kb * 8 + q];
      *reinterpret_cast<uint4*>(smem + cfg.off_b + (uint32_t)(v * KB + kb) * btile + wg::sw128_chunk(r, q)) = val;
    }
    // ||c_j||^2 from the pack's exact 3-way split [hi, mid, lo] (hi + mid + lo == the fp32 value)
    const float* bcn = reinterpret_cast<const float*>(a.pack + a.L.off_bcn2);
    for (int j = tid; j < N; j += T2_THREADS) {
      float v = 3.0e38f;
      if (j < NS) { const int jg = slice * NS + j; const float* p = bcn + (jg >> 3) * 64 + (jg & 7) * 4; v = (p[0] + p[1]) + p[2]; }
      cn_s[j] = v;
    }
    wg::fence_proxy_async();                                 // generic-proxy stores -> visible to wgmma
  }
  __syncthreads();

  const long long ntiles = (a.n + T2_BM - 1) / T2_BM;
  const long long my_tiles = group < ntiles ? (ntiles - group + cfg.G - 1) / cfg.G : 0;
  const long long npairs = (my_tiles + 1) / 2;              // warpgroup w takes the group's tiles 2p + w
  const __nv_bfloat16* X = reinterpret_cast<const __nv_bfloat16*>(a.X);
  const uint32_t xs_u32 = sbase + cfg.off_x + (uint32_t)wgi * 2u * stage_bytes;
  const int nq = KB * 8;
  auto load_tile = [&](long long p, int stage) {
    const long long lt = 2 * p + wgi;
    if (lt < my_tiles) {
      const long long row0 = (group + lt * cfg.G) * T2_BM;
      for (int i = t; i < T2_BM * nq; i += 128) {
        const int r = i / nq, rem = i - r * nq, kb = rem >> 3, q = rem & 7;
        const int col = kb * 64 + q * 8;
        const long long row = row0 + r;
        const int bytes = (row < a.n && col < d) ? min(16, (d - col) * 2) : 0;
        wg::cp16(xs_u32 + (uint32_t)stage * stage_bytes + (uint32_t)kb * xkblk + wg::sw128_chunk(r, q),
                 bytes ? X + row * a.ldx + col : X, bytes);
      }
    }
    wg::cp_commit();
  };

  const int rA = wq * 16 + (lane >> 2);                      // this thread's accumulator rows: rA, rA + 8
  const uint64_t db0 = wg::desc_sw128(sbase + cfg.off_b);
  const float cnmax = (float)reinterpret_cast<const PackHeader*>(a.pack)->cn_max;

  load_tile(0, 0);
#pragma unroll 1
  for (long long p = 0; p < npairs; ++p) {
    const int stage = (int)(p & 1);
    load_tile(p + 1, stage ^ 1);
    wg::cp_wait1();
    wg::wg_sync(1 + wgi);                                    // tile p is in shared memory (every thread's copies)
    const long long lt = 2 * p + wgi;
    if (lt < my_tiles) {
      const long long row0 = (group + lt * cfg.G) * T2_BM;
      const uint32_t xs = xs_u32 + (uint32_t)stage * stage_bytes;
      // ---- acc = X . Bhi^T + X . Blo^T ----
      float acc[N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
      wg::fence();
#pragma unroll 1
      for (int ks = 0; ks < cfg.KS; ++ks) {
        // K-block kb: A tile 8 KB further, B tile `btile` further; K-step kq: 32 bytes inside the swizzle atom
        const int kb = ks >> 2, kq = ks & 3;
        const uint64_t da = wg::desc_sw128(xs + (uint32_t)kb * xkblk) + (uint64_t)(2 * kq);
        const uint64_t boff = (uint64_t)(((uint32_t)kb * btile) >> 4) + (uint64_t)(2 * kq);
        wg::Mma<N>::ss_bf16(acc, da, db0 + boff, ks > 0);
        wg::Mma<N>::ss_bf16(acc, da, db0 + (uint64_t)(((uint32_t)KB * btile) >> 4) + boff, 1);
      }
      wg::commit();
      // ---- row norms ||x||^2 while the MMAs run: thread (row r, half of the 16-byte chunks) ----
      {
        const int r = t & 63, part = t >> 6;
        float s0 = 0.f, s1 = 0.f;
        for (int j = part; j < nq; j += 2) {
          const uint4 v = *reinterpret_cast<const uint4*>(smem + (xs - sbase) + (uint32_t)(j >> 3) * xkblk + wg::sw128_chunk(r, j & 7));
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            // two bf16 per word: the low half is the lower element
            const float lo = __uint_as_float(w[e] << 16), hi = __uint_as_float(w[e] & 0xffff0000u);
            s0 = fmaf(lo, lo, s0);
            s1 = fmaf(hi, hi, s1);
          }
        }
        xn_s[part * T2_BM + r] = s0 + s1;
      }
      wg::wait_all();
      wg::pin(acc);
      wg::wg_sync(1 + wgi);                                  // xn_s complete

      // ---- arg-min, near-tie test (bound = tau (||x||^2 + max ||c||^2): the accumulator holds ||c||^2 - 2 x.c) ----
      wg::Best2 b0, b1;
      wg::tile_best2<N>(acc, cn_s, lane, b0, b1);
      if ((lane & 3) == 0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const wg::Best2 b = h ? b1 : b0;
          const int r = rA + 8 * h;
          const long long row = row0 + r;
          if (row >= a.n) continue;
          const float xn = xn_s[r] + xn_s[T2_BM + r];
          const bool out_of_range = !(xn < 3.0e38f);
          const bool tie = !(b.m2 > b.m1 + a.tau * (xn + cnmax)) || out_of_range;
          const int bj = slice * NS + ((tie || b.j >= NS) ? 0 : b.j);
          if (S == 1) {
            if (!(tie && a.k > 1)) {
              if (a.labels) a.labels[row] = bj;
            } else {
              const int slot = atomicAdd(a.defer_cnt, 1);
              a.defer_idx[slot] = (int)row;
            }
          } else {
            // partial record of this (slice, row): slice minimum, label or -1 (near-tie inside the slice), ||x||^2
            a.rec[(size_t)slice * a.n + row] = make_float4(b.m1, b.m2, __int_as_float(tie ? -1 : bj), xn);
          }
        }
      }
    }
    wg::wg_sync(1 + wgi);                                    // the stage and xn_s may be refilled
  }
}

// ------------------------------------------------------------------------------------------
// S > 1: fold the S partial records of every row.  The slice holding the smallest minimum gives the label unless that
// slice saw a near-tie itself or another slice's minimum is within the rounding bound: those rows go to the float64
// re-check like on every other path.  Exactly equal minima in two slices are a near-tie by construction.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
tc2_combine_kernel(ChunkArgs a, int S) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  const PackHeader* hdr = reinterpret_cast<const PackHeader*>(a.pack);
  const float cnmax = (float)hdr->cn_max;
  for (long long row = blockIdx.x * (long long)blockDim.x + threadIdx.x; row < a.n; row += (long long)gridDim.x * blockDim.x) {
    float best = CUDART_INF_F, second = CUDART_INF_F, xn = 0.f;
    int lab = -1;
    for (int s = 0; s < S; ++s) {
      const float4 r = a.rec[(size_t)s * a.n + row];
      xn = r.w;
      if (r.x < best) { second = best; best = r.x; lab = __float_as_int(r.z); }
      else second = fminf(second, r.x);
    }
    const float bound = a.tau * (xn + cnmax);
    const bool flagged = (lab < 0 || !(second - best > bound) || !(xn < 3.0e38f)) && a.k > 1;
    if (!flagged) {
      if (a.labels) a.labels[row] = lab < 0 ? 0 : lab;
    } else {
      const int slot = atomicAdd(a.defer_cnt, 1);
      a.defer_idx[slot] = (int)row;
    }
  }
}

// ------------------------------------------------------------------------------------------
// float64 re-check of the deferred rows (labels only: distances and sums of these shapes come from the row passes).
// Same form as the reference's float64 E-step (scikit-learn ArgKmin: ||c||^2 - 2 x.c, the row norm is common to all
// centres): one DFMA per (row, centre, feature).  Thread j <-> centres j, j + 256, ...; float64 centres transposed
// [d][kp2] (coalesced reads, L2-resident: every group of rows streams the whole [d][k] block from L2, so 16 rows share
// one pass); the group's rows are staged as float64 in shared memory (broadcast reads).
// ------------------------------------------------------------------------------------------
static const int R2_ROWS = 16;

template <typename TX>
__device__ __forceinline__ float ld_as_float(const TX* p);
template <> __device__ __forceinline__ float ld_as_float<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

template <typename TX>
__global__ void __launch_bounds__(256)
tc2_recheck_kernel(ChunkArgs a, int kp2) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  __shared__ double xs[128][R2_ROWS];            // [feature][row]: the rows of a feature are one 128-byte broadcast
  __shared__ double wd[R2_ROWS][8];
  __shared__ int wj[R2_ROWS][8];
  __shared__ long long rows_s[R2_ROWS];
  const unsigned int abort_code = *reinterpret_cast<const volatile unsigned int*>(a.defer_cnt + 1);
  if (blockIdx.x == 0 && threadIdx.x == 0 && abort_code) {
    // a pipeline wait of the tensor kernel timed out: make that loud (NaN cost / sums, negative label)
    if (a.out_sums) a.out_sums[0] = CUDART_NAN;
    if (a.out_dist_sum) *a.out_dist_sum = CUDART_NAN;
    if (a.labels && a.n > 0) a.labels[0] = -1;
  }
  const int cnt = *a.defer_cnt;
  if ((int)blockIdx.x * R2_ROWS >= cnt) return;
  const int k = a.k, d = a.d, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const double* gT = reinterpret_cast<const double*>(a.pack + a.L.off_c64T2);
  const double* cn64 = reinterpret_cast<const double*>(a.pack + a.L.off_cn64);
  const TX* X = reinterpret_cast<const TX*>(a.X);
  for (int f0 = blockIdx.x * R2_ROWS; f0 < cnt; f0 += gridDim.x * R2_ROWS) {
    const int nr = min(R2_ROWS, cnt - f0);
    __syncthreads();
    if (tid < R2_ROWS) rows_s[tid] = tid < nr ? (long long)a.defer_idx[f0 + tid] : -1;
    __syncthreads();
    for (int e = tid; e < R2_ROWS * 128; e += 256) {
      const int r = e >> 7, i = e & 127;
      xs[i][r] = (r < nr && i < d) ? (double)ld_as_float<TX>(X + rows_s[r] * a.ldx + i) : 0.0;
    }
    __syncthreads();
    double bd[R2_ROWS];
    int bj[R2_ROWS];
#pragma unroll
    for (int r = 0; r < R2_ROWS; ++r) { bd[r] = CUDART_INF; bj[r] = 0x7fffffff; }
    for (int j = tid; j < k; j += 256) {
      double s0[R2_ROWS];
#pragma unroll
      for (int r = 0; r < R2_ROWS; ++r) s0[r] = 0.0;
#pragma unroll 4
      for (int i = 0; i < d; ++i) {
        const double c0 = gT[(size_t)i * kp2 + j];
#pragma unroll
        for (int r = 0; r < R2_ROWS; ++r) s0[r] = fma(xs[i][r], c0, s0[r]);
      }
      const double cn = cn64[j];
#pragma unroll
      for (int r = 0; r < R2_ROWS; ++r) {
        const double dist = fma(-2.0, s0[r], cn);            // + ||x||^2 is common to all centres of the row
        if (dist < bd[r]) { bd[r] = dist; bj[r] = j; }      // ascending j: the lowest index wins exact ties
      }
    }
#pragma unroll
    for (int r = 0; r < R2_ROWS; ++r) {
      double vd = bd[r];
      int vj = bj[r];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const double od = __shfl_xor_sync(0xffffffffu, vd, o);
        const int oj = __shfl_xor_sync(0xffffffffu, vj, o);
        if (od < vd || (od == vd && oj < vj)) { vd = od; vj = oj; }
      }
      if (lane == 0) { wd[r][wid] = vd; wj[r][wid] = vj; }
    }
    __syncthreads();
    if (tid < nr) {
      const int r = tid;
      double fd = wd[r][0];
      int fj = wj[r][0];
      for (int w = 1; w < 8; ++w) if (wd[r][w] < fd || (wd[r][w] == fd && wj[r][w] < fj)) { fd = wd[r][w]; fj = wj[r][w]; }
      if (a.labels) a.labels[rows_s[r]] = fj == 0x7fffffff ? 0 : fj;
    }
  }
}


// ------------------------------------------------------------------------------------ host
static bool make_cfg2(int d, int k, int sm_count, Tc2Cfg* c) {
  const Tc2Geom g = tc2_geom(k, d);
  c->S = g.S; c->NS = g.NS; c->KB = g.KB; c->KS = (d + 15) / 16;
  if (g.S > sm_count) return false;
  c->G = sm_count / g.S;
  const uint32_t N = (uint32_t)wg::mma_n(g.NS);
  uint32_t o = 0;
  c->off_b = o; o += 2u * (uint32_t)g.KB * N * 128u;                 // (hi, lo) x K-blocks of the slice
  c->off_x = o; o += 2u * 2u * (uint32_t)g.KB * T2_BM * 128u;        // 2 warpgroups x 2 stages
  c->off_cn = o; o += N * 4u;
  c->off_xn = o; o += 2u * 2u * T2_BM * 4u;
  c->total = o;
  return o <= 227u * 1024u;
}

template <int N>
static int launch_assign(const ChunkArgs& a, const Tc2Cfg& cfg, cudaStream_t s) {
  BKM_CUDA_TRY(cudaFuncSetAttribute(tc2_assign_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cfg.total));
  tc2_assign_kernel<N><<<cfg.G * cfg.S, T2_THREADS, cfg.total, s>>>(a, cfg);
  return 0;
}

// E-step of one chunk on the large-shape tensor path; the M-step / distances follow as row passes (bkm_rowpass.cu).
// *grid_out: number of partial slots the row passes wrote (for reduce_partials), 0 when there is nothing to reduce.
int launch_tc2(const ChunkArgs& a0, bool mstep, int sm_count, int* grid_out, cudaStream_t s) {
  ChunkArgs a = a0;
  if (!tc2_shape(a.d, a.k, BKM_BF16)) return BKM_EUNSUPPORTED;
  if ((reinterpret_cast<uintptr_t>(a.X) & 15) || (a.ldx % 8)) return BKM_EALIGN;     // 16-byte staging copies
  Tc2Cfg cfg;
  if (!make_cfg2(a.d, a.k, sm_count, &cfg)) return BKM_EUNSUPPORTED;
  const Tc2Geom g = tc2_geom(a.k, a.d);
  const long long ntiles = (a.n + T2_BM - 1) / T2_BM;
  if (ntiles < cfg.G) cfg.G = (int)ntiles;
  if (cfg.G < 1) cfg.G = 1;
  BKM_CUDA_TRY(cudaMemsetAsync(a.defer_cnt, 0, 2 * sizeof(int), s));          // [0] deferred rows, [1] abort word
  int rc;
  switch (wg::mma_n(cfg.NS)) {
    case 16: rc = launch_assign<16>(a, cfg, s); break;
    case 32: rc = launch_assign<32>(a, cfg, s); break;
    case 64: rc = launch_assign<64>(a, cfg, s); break;
    case 128: rc = launch_assign<128>(a, cfg, s); break;
    default: rc = launch_assign<256>(a, cfg, s); break;
  }
  if (rc) return rc;
  note_launch(2);
  BKM_CUDA_TRY(cudaGetLastError());
  if (cfg.S > 1) {
    long long nb = (a.n + 255) / 256;
    if (nb > sm_count * 8) nb = sm_count * 8;
    tc2_combine_kernel<<<(int)nb, 256, 0, s>>>(a, cfg.S);
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
  }
  if (a.k > 1) {
    tc2_recheck_kernel<__nv_bfloat16><<<sm_count * 4, 256, 0, s>>>(a, g.kp2);
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
  }
  // label-indexed row passes
  int parts = 0;
  const bool want_dist = a.min_out != nullptr || a.want_sum;
  if (want_dist) {
    rc = launch_rowpass_dist(a, BKM_BF16, sm_count, &parts, s);
    if (rc) return rc;
  }
  int mparts = 0;
  if (mstep) {
    rc = launch_rowpass_mstep(a, BKM_BF16, sm_count, &mparts, s);
    if (rc) return rc;
  }
  // encode both partial counts for reduce_partials: low 16 bits = sums/count parts, high bits = distance parts
  *grid_out = (mparts & 0xffff) | (parts << 16);
  return 0;
}

}  // namespace bkm

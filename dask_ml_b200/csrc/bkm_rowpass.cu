// bkm_rowpass.cu — label-indexed row passes for shapes whose k x d partial sums do not fit one CTA (the large-shape
// tensor path, bkm_tc2.cu: BASELINE config C5, k = 1024, d = 128 -> 512 KB of fp32 sums).
//
//   rowpass_mstep_kernel   M-step (_centers_dense, dask_ml/cluster/k_means.py:572-582 + da.bincount :548) from the
//                          labels the E-step wrote: the CLUSTERS are cut into DS interleaved slices so that the
//                          (k / DS) x d fp32 sums of a slice DO fit shared memory; CTA (row block rb, cluster slice cs)
//                          scans the labels of its rows and gathers the rows of its clusters (whole rows, coalesced:
//                          every row of X is read once over the DS CTAs), warp w owning the local clusters
//                          (c / DS) % NW == w (no atomics, fixed order).  Per-row-block partials are folded in
//                          float64 by reduce_partials in row-block order.
//   rowpass_dist_kernel    winning distance sum_i (x_i - c_label,i)^2 in direct form (fp32, no cancellation), one warp per
//                          row: min_out and the per-CTA distance sums (inertia, k_means.py:566 / k-means|| cost :466-469).
// The tensor-bound E-step dominates these shapes (C5: 22.6 ms at the tensor roof vs 5 ms for a sweep of X at the HBM
// roof), so the extra sweep costs ~1/5 of an iteration; shapes whose sums fit a CTA keep the fused kernels.
#include "bkm_common.cuh"
#include "bkm_ptx.cuh"
#include <cuda_bf16.h>
#include <math_constants.h>

namespace bkm {

static const int RP_THREADS = 512;
static const int RP_NW = RP_THREADS / 32;
static const int RP_TILE = 4096;              // rows per binning tile (row offsets inside a tile take 12 bits)
static const int RP_BATCH = 16;               // rows gathered per batch (loads in flight per warp)
static const int RP_MAXB = 256;               // buckets = cluster slices x warps (CS <= 16)

template <typename TX> __device__ __forceinline__ float rp_to_float(TX v);
template <> __device__ __forceinline__ float rp_to_float<float>(float v) { return v; }
template <> __device__ __forceinline__ float rp_to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

struct RpCfg {
  int CS, LCS, RB, KL;     // cluster slices (a power of two, LCS = log2), row blocks (grid = RB * CS), clusters per slice
  int NB;                  // buckets = CS * NW
  long long ntiles, tiles_per_block;
  uint32_t off_sums, off_cnt, total;
};

// FPL features per lane of a row: a warp reads a whole row with one load per lane (lane l: features l*FPL ...).
// raw = the loaded bits (kept packed while the loads of a batch are in flight), add() widens and accumulates
template <typename TX, int FPL> struct RowPiece;
// (volatile asm loads: the compiler must not sink a load next to its use — the point is 16 rows in flight per warp)
template <> struct RowPiece<__nv_bfloat16, 1> {
  unsigned short raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { asm volatile("ld.global.nc.u16 %0, [%1];" : "=h"(raw) : "l"(p)); }
  __device__ __forceinline__ void add(float* sr) const { sr[0] += __uint_as_float((uint32_t)raw << 16); }
};
template <> struct RowPiece<__nv_bfloat16, 2> {
  uint32_t raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) { asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(raw) : "l"(p)); }
  __device__ __forceinline__ void add(float* sr) const {
    float2 t = *reinterpret_cast<float2*>(sr);
    t.x += __uint_as_float(raw << 16); t.y += __uint_as_float(raw & 0xffff0000u);
    *reinterpret_cast<float2*>(sr) = t;
  }
};
template <> struct RowPiece<__nv_bfloat16, 4> {
  uint2 raw;
  __device__ __forceinline__ void load(const __nv_bfloat16* p) {
    asm volatile("ld.global.nc.v2.u32 {%0, %1}, [%2];" : "=r"(raw.x), "=r"(raw.y) : "l"(p));
  }
  __device__ __forceinline__ void add(float* sr) const {
    float4 t = *reinterpret_cast<float4*>(sr);             // one 16-byte access per lane: conflict-free
    t.x += __uint_as_float(raw.x << 16); t.y += __uint_as_float(raw.x & 0xffff0000u);
    t.z += __uint_as_float(raw.y << 16); t.w += __uint_as_float(raw.y & 0xffff0000u);
    *reinterpret_cast<float4*>(sr) = t;
  }
};

// ------------------------------------------------------------------------------------------
// Step 1: bin the rows of every 4096-row tile by bucket = (cluster slice, owner warp) of their label — a stable
// counting sort per tile (rows of a bucket stay in row order, so the sums are reproducible).  bins[tile*4096 + pos]
// = row-in-tile | local cluster << 12; tile_off[tile][b] = first position of bucket b, [NB] = valid rows of the tile.
// One CTA per tile (grid-stride); labels are read once.
// ------------------------------------------------------------------------------------------
// The owner warp of a cluster inside its slice comes from the BALANCE TABLE when the previous chunk call left one for
// this (k, CS) (rowpass_balance_kernel: clusters ranked by size and dealt to the 16 warps in snake order), else it is
// (c / CS) % NW.  Cluster sizes are heavy-tailed (a centre that covers five blobs owns 5x the mean) and a CTA runs as
// long as its most loaded warp: 1.25-1.45x the mean with the static map.  The table only moves clusters between warps;
// the rows of a cluster are still added in row order by ONE warp, so the sums are bit-identical with or without it.
static const unsigned RP_BAL_MAGIC = 0x62616c31u;     // "bal1"

__global__ void __launch_bounds__(RP_THREADS)
rowpass_bin_kernel(const int* __restrict__ labels, long long n, RpCfg c, unsigned* __restrict__ bins, int* __restrict__ tile_off,
                   const unsigned char* __restrict__ bal, int k, const int* skip) {
  if (skip && *skip) return;
  const unsigned* bh = reinterpret_cast<const unsigned*>(bal);
  const bool use_bal = bal && bh[0] == RP_BAL_MAGIC && bh[1] == (unsigned)k && bh[2] == (unsigned)c.CS;
  const unsigned char* btab = bal + 16;
  __shared__ int cntw[RP_NW][RP_MAXB];          // pass 1: rows of (warp, bucket); pass 2: running write position
  __shared__ int base_s[RP_MAXB + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int NB = c.NB;
  const unsigned lt_mask = (1u << lane) - 1u;
  for (long long t = blockIdx.x; t < c.ntiles; t += gridDim.x) {
    const long long r0 = t * RP_TILE;
    __syncthreads();
    for (int i = tid; i < RP_NW * RP_MAXB; i += RP_THREADS) (&cntw[0][0])[i] = 0;
    __syncthreads();
    int bk[8], cl[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {                 // warp w bins rows [w*256, w*256 + 256) of the tile, 8 groups of 32
      const long long r = r0 + warp * 256 + u * 32 + lane;
      const int ml = r < n ? __ldg(labels + r) : -1;
      cl[u] = ml >> c.LCS;
      int ow = cl[u] & (RP_NW - 1);
      if (use_bal && ml >= 0) ow = min((int)btab[ml], RP_NW - 1);
      bk[u] = ml < 0 ? -1 : ((ml & (c.CS - 1)) * RP_NW + ow);
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const unsigned same = __match_any_sync(0xffffffffu, bk[u]);
      if (bk[u] >= 0 && (same & lt_mask) == 0) cntw[warp][bk[u]] += __popc(same);     // the group's first lane
      __syncwarp();
    }
    __syncthreads();
    // exclusive prefix: buckets in order, warps in order inside a bucket
    if (tid < NB) {
      int tot = 0;
      for (int w = 0; w < RP_NW; ++w) tot += cntw[w][tid];
      base_s[tid + 1] = tot;
    }
    if (tid == 0) base_s[0] = 0;
    __syncthreads();
    if (tid == 0) for (int b = 0; b < NB; ++b) base_s[b + 1] += base_s[b];
    __syncthreads();
    if (tid < NB) {
      int pos = base_s[tid];
      for (int w = 0; w < RP_NW; ++w) { const int cur = cntw[w][tid]; cntw[w][tid] = pos; pos += cur; }
    }
    for (int b = tid; b <= NB; b += RP_THREADS) tile_off[t * (RP_MAXB + 1) + b] = base_s[b];
    __syncthreads();
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const unsigned same = __match_any_sync(0xffffffffu, bk[u]);
      int pos = 0;
      if (bk[u] >= 0) {
        const int leader = __ffs(same) - 1;
        if (lane == leader) { pos = cntw[warp][bk[u]]; cntw[warp][bk[u]] = pos + __popc(same); }
        pos = __shfl_sync(same, pos, leader) + __popc(same & lt_mask);
        bins[r0 + pos] = (unsigned)(warp * 256 + u * 32 + lane) | ((unsigned)cl[u] << 12);
      }
      __syncwarp();
    }
  }
}

// ------------------------------------------------------------------------------------------
// Step 3 (after the M-step): rebuild the balance table from THIS call's per-cluster counts for the next call.
// Block cs ranks the KL clusters of its slice by size (ties by index) and deals rank r to warp r % 16 on even rounds,
// 15 - r % 16 on odd rounds.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
rowpass_balance_kernel(const int* __restrict__ pcnt, int parts, int k, RpCfg c, unsigned char* bal, const int* skip) {
  if (skip && *skip) return;
  extern __shared__ int sz_s[];                    // [KL]
  const int cs = blockIdx.x, CS = c.CS, KL = c.KL;
  for (int i = threadIdx.x; i < KL; i += blockDim.x) {
    const int cg = i * CS + cs;
    int t = 0;
    if (cg < k) for (int p = 0; p < parts; ++p) t += pcnt[(size_t)p * k + cg];
    sz_s[i] = t;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < KL; i += blockDim.x) {
    const int cg = i * CS + cs;
    if (cg >= k) continue;
    const int mine = sz_s[i];
    int rank = 0;
    for (int j = 0; j < KL; ++j) rank += (sz_s[j] > mine || (sz_s[j] == mine && j < i)) ? 1 : 0;
    const int r = rank & (RP_NW - 1);
    bal[16 + cg] = (unsigned char)(((rank / RP_NW) & 1) ? RP_NW - 1 - r : r);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    unsigned* bh = reinterpret_cast<unsigned*>(bal);
    bh[0] = RP_BAL_MAGIC; bh[1] = (unsigned)k; bh[2] = (unsigned)CS; bh[3] = 0u;
  }
}

// ------------------------------------------------------------------------------------------
// Step 2: the M-step proper.  CTA (row block rb, cluster slice cs) owns the clusters c with c % CS == cs (KL of them:
// their k/CS x d fp32 sums fit shared memory); warp w owns the local clusters (c / CS) % NW == w, i.e. bucket
// cs * NW + w.  It walks its bucket's entries tile by tile (coalesced reads of the bin list) and GATHERS the rows,
// whole rows, one coalesced load per warp and row, 16 loads in flight before the first one is consumed; rows are added
// into the warp's clusters with plain read-add-write on shared memory (no atomics, row order: reproducible).
// Every row of X is read exactly once over the CS CTAs of a row block; no label is scanned twice.
// ------------------------------------------------------------------------------------------
template <typename TX, int FPL>
__global__ void __launch_bounds__(RP_THREADS, 1)
rowpass_mstep_kernel(ChunkArgs a, RpCfg c, const unsigned* __restrict__ bins, const int* __restrict__ tile_off) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  extern __shared__ __align__(128) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int k = a.k, d = a.d, CS = c.CS;
  const int rb = blockIdx.x / CS, cs = blockIdx.x % CS;
  constexpr int RW = 32 * FPL;                                       // floats per cluster row in shared memory
  float* sums_s = reinterpret_cast<float*>(smem + c.off_sums);       // [KL][RW]
  int* cnts_s = reinterpret_cast<int*>(smem + c.off_cnt);            // [KL]
  const TX* X = reinterpret_cast<const TX*>(a.X);
  for (int i = tid; i < c.KL * RW; i += RP_THREADS) sums_s[i] = 0.f;
  for (int i = tid; i < c.KL; i += RP_THREADS) cnts_s[i] = 0;
  __syncthreads();

  const long long t0 = (long long)rb * c.tiles_per_block;
  const long long t1 = min(c.ntiles, t0 + c.tiles_per_block);
  const int bucket = cs * RP_NW + warp;
  const bool lane_on = lane * FPL < d;                               // this lane's piece holds real features
  // Software pipeline: while the 16 rows of batch i are in flight, the entries of batch i + 1 (and the bucket bounds of
  // the next tile) are already being fetched, so a batch costs ONE memory round trip.
  long long t = t0;
  int hi = 0, e0 = 0, nlo = 0, nhi = 0;
  if (t0 < t1) {
    e0 = __ldg(tile_off + t0 * (RP_MAXB + 1) + bucket);
    hi = __ldg(tile_off + t0 * (RP_MAXB + 1) + bucket + 1);
    if (t0 + 1 < t1) {
      nlo = __ldg(tile_off + (t0 + 1) * (RP_MAXB + 1) + bucket);
      nhi = __ldg(tile_off + (t0 + 1) * (RP_MAXB + 1) + bucket + 1);
    }
  }
  unsigned mine_n = 0u;
  int nb_n = 0;
  long long r0_n = 0;
  auto advance = [&]() -> bool {            // warp-uniform: queue the next non-empty batch and issue its entry load
    if (t >= t1) return false;
    while (e0 >= hi) {
      if (++t >= t1) return false;
      e0 = nlo; hi = nhi;
      if (t + 1 < t1) {
        nlo = __ldg(tile_off + (t + 1) * (RP_MAXB + 1) + bucket);
        nhi = __ldg(tile_off + (t + 1) * (RP_MAXB + 1) + bucket + 1);
      }
    }
    nb_n = min(RP_BATCH, hi - e0);
    r0_n = t * RP_TILE;
    mine_n = lane < nb_n ? __ldg(bins + r0_n + e0 + lane) : 0u;
    e0 += RP_BATCH;
    return true;
  };
  bool have = advance();
#pragma unroll 1
  while (have) {
    const unsigned mine = mine_n;
    const int nb = nb_n;
    const long long r0 = r0_n;
    have = advance();
    RowPiece<TX, FPL> x[RP_BATCH];
    int cc[RP_BATCH];
    const unsigned e_first = __shfl_sync(0xffffffffu, mine, 0);
#pragma unroll
    for (int q = 0; q < RP_BATCH; ++q) {
      const unsigned e = __shfl_sync(0xffffffffu, mine, q);
      cc[q] = (int)(e >> 12);
      // rows past the batch re-load its first row (never used): the loads stay unconditional and back to back
      const unsigned eq = q < nb ? e : e_first;
      if (lane_on) x[q].load(X + (r0 + (long long)(eq & 0xfffu)) * a.ldx + lane * FPL);
    }
    __syncwarp();                                                    // all loads of the batch are issued before the first use
#pragma unroll
    for (int q = 0; q < RP_BATCH; ++q) {
      if (q < nb) {
        if (lane_on) x[q].add(sums_s + (size_t)cc[q] * RW + lane * FPL);
        if (lane == 0) cnts_s[cc[q]] += 1;
      }
    }
  }
  __syncthreads();
  // ---- flush: local cluster cl is cluster cl * CS + cs ----
  float* g = reinterpret_cast<float*>(a.psum) + (size_t)rb * k * d;
  for (int i = tid; i < c.KL * RW; i += RP_THREADS) {
    const int cl = i / RW, f = i - cl * RW;
    const int cg = cl * CS + cs;
    if (cg < k && f < d) g[(size_t)cg * d + f] = sums_s[i];
  }
  int* gc = a.pcnt + (size_t)rb * k;
  for (int i = tid; i < c.KL; i += RP_THREADS) {
    const int cg = i * CS + cs;
    if (cg < k) gc[cg] = cnts_s[i];
  }
}

template <typename TX>
__global__ void __launch_bounds__(256)
rowpass_dist_kernel(ChunkArgs a) {
  if (a.skip && *a.skip) return;                            // converged loop: no-op iteration

  __shared__ double red_s[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int d = a.d, d4 = a.L.d4;
  const TX* X = reinterpret_cast<const TX*>(a.X);
  const float* gC = reinterpret_cast<const float*>(a.pack + a.L.off_cT);        // fp32 centres [k][d4]
  double dsum = 0.0;
  const long long gw = (long long)blockIdx.x * 8 + warp, nw = (long long)gridDim.x * 8;
  for (long long row = gw; row < a.n; row += nw) {
    const int lbl = a.labels[row];
    const TX* xr = X + row * a.ldx;
    const float* cr = gC + (size_t)(lbl < 0 ? 0 : lbl) * d4;
    // float64: (x - c)^2 of bf16 rows leaves fp32's range at either end of it (|x| beyond 2^64 or below 2^-63)
    double sacc = 0.0;
    for (int i = lane; i < d; i += 32) {
      const double df = (double)rp_to_float<TX>(xr[i]) - (double)cr[i];
      sacc = fma(df, df, sacc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
    if (lane == 0) {
      const double outv = a.squared ? sacc : sqrt(sacc);
      dsum += outv;
      if (a.min_out) reinterpret_cast<float*>(a.min_out)[row] = (float)outv;
    }
  }
  if (lane == 0) red_s[warp] = dsum;
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red_s[w];
    a.pin[blockIdx.x] = t;
  }
}

static bool make_rp_cfg(int k, int d, int sm_count, int psum_slots, long long n, RpCfg* c, int* fpl_out) {
  const Tc2Geom g = tc2_geom(k, d);
  const int fpl = d <= 32 ? 1 : (d <= 64 ? 2 : 4);
  *fpl_out = fpl;
  c->CS = g.DS;                                       // cluster slices (geometry shared with the workspace sizing)
  c->LCS = 0;
  while ((1 << c->LCS) < c->CS) ++c->LCS;
  c->NB = c->CS * RP_NW;
  if (c->NB > RP_MAXB) return false;
  c->KL = (k + c->CS - 1) / c->CS;
  c->ntiles = (n + RP_TILE - 1) / RP_TILE;
  int rb = sm_count / c->CS;
  if (rb < 1) rb = 1;
  if (rb > psum_slots) rb = psum_slots;
  if (rb > c->ntiles) rb = (int)(c->ntiles > 0 ? c->ntiles : 1);
  c->tiles_per_block = (c->ntiles + rb - 1) / rb;
  rb = (int)((c->ntiles + c->tiles_per_block - 1) / c->tiles_per_block);     // no empty row blocks
  c->RB = rb;
  uint32_t o = 0;
  c->off_sums = o; o += (uint32_t)c->KL * 32u * fpl * 4u;
  c->off_cnt = o; o += (uint32_t)align_up((size_t)c->KL * 4, 16);
  c->total = o;
  return o <= 227 * 1024;
}

// binning: one CTA per 4096-row tile, grid-strided past 4 CTAs per SM
static int bin_grid(const RpCfg& c, int sm_count) {
  return (int)(c.ntiles < (long long)sm_count * 4 ? c.ntiles : (long long)sm_count * 4);
}
// distances: one warp per row, grid-strided past 8 CTAs per SM (and the partial slots)
static int dist_grid(long long n, int sm_count, int part_slots) {
  long long grid = (n + 7) / 8;
  if (grid > (long long)sm_count * 8) grid = (long long)sm_count * 8;
  if (grid > part_slots) grid = part_slots;
  return (int)(grid < 1 ? 1 : grid);
}

int launch_rowpass_mstep(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s) {
  if (!a.labels) return BKM_EINVAL;                     // the row pass is driven by the labels
  if (x_dtype != BKM_BF16) return BKM_EDTYPE;
  RpCfg c;
  int fpl = 0;
  if (!make_rp_cfg(a.k, a.d, sm_count, a.psum_slots, a.n, &c, &fpl)) return BKM_EUNSUPPORTED;
  unsigned* bins = reinterpret_cast<unsigned*>(a.bin_list);
  int* tile_off = a.bin_off;
  rowpass_bin_kernel<<<bin_grid(c, sm_count), RP_THREADS, 0, s>>>(a.labels, a.n, c, bins, tile_off, a.k <= 4096 ? a.bal : nullptr, a.k, a.skip);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
#define RP_GO(F)                                                                                                   \
  {                                                                                                                \
    auto kern = rowpass_mstep_kernel<__nv_bfloat16, F>;                                                            \
    BKM_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.total));           \
    kern<<<c.RB * c.CS, RP_THREADS, c.total, s>>>(a, c, bins, tile_off);                                           \
  }
  if (fpl == 1) RP_GO(1) else if (fpl == 2) RP_GO(2) else RP_GO(4)
#undef RP_GO
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  if (a.bal && a.k <= 4096) {
    rowpass_balance_kernel<<<c.CS, 1024, (size_t)c.KL * sizeof(int), s>>>(a.pcnt, c.RB, a.k, c, a.bal, a.skip);
    note_launch();
    BKM_CUDA_TRY(cudaGetLastError());
  }
  *parts_out = c.RB;
  return 0;
}

int launch_rowpass_dist(const ChunkArgs& a, int x_dtype, int sm_count, int* parts_out, cudaStream_t s) {
  if (!a.labels) return BKM_EINVAL;
  const int grid = dist_grid(a.n, sm_count, a.part_slots);
  if (x_dtype == BKM_BF16) rowpass_dist_kernel<__nv_bfloat16><<<(int)grid, 256, 0, s>>>(a);
  else rowpass_dist_kernel<float><<<(int)grid, 256, 0, s>>>(a);
  note_launch();
  BKM_CUDA_TRY(cudaGetLastError());
  *parts_out = grid;
  return 0;
}

// bkm_debug_tc2_layout's row-pass half: {DS (= CS), NB, KL, RB, tiles_per_block, bin grid, dist grid, FPL, mstep
// shared-memory bytes} of an n-row call with the workspace ws_layout sizes for sm_count SMs
int rowpass_layout(int k, int d, long long n, int sm_count, int* out) {
  const WsLayout W = ws_layout(n, d, k, BKM_BF16, sm_count);
  RpCfg c;
  int fpl = 0;
  if (!make_rp_cfg(k, d, sm_count, W.psum_slots, n, &c, &fpl)) return BKM_EUNSUPPORTED;
  out[0] = c.CS;
  out[1] = c.NB;
  out[2] = c.KL;
  out[3] = c.RB;
  out[4] = (int)c.tiles_per_block;
  out[5] = bin_grid(c, sm_count);
  out[6] = dist_grid(n, sm_count, W.part_slots);
  out[7] = fpl;
  out[8] = (int)c.total;
  return 0;
}

}  // namespace bkm

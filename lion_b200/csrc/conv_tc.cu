// lion_b200 -- tensor-core convolution for sm_90a: wgmma (TF32, FP32 accumulators in registers), operands staged by
// cp.async.bulk + mbarrier pipelines, warp-specialised.
//
// One kernel serves the 3x3x3 voxel convolutions (reference: nn.Conv3d in
// models/pvcnn2_ada.py:211-222 -> cuDNN, 98 % of the step's FLOPs) and the 1x1 point
// convolutions (SharedMLP / attention projections, pvcnn2_ada.py:125-137, :51-52).
//
// Formulation (im2col-free implicit GEMM on the zero-haloed packed layouts, see
// packed_kernels.cuh):  out[p][co] = sum_tap sum_ci in[p + off(tap)][ci] * W[tap][ci][co].
//   * M = 64 rows per wgmma, one block per consumer warpgroup; N = output channels (<= 128 per CTA), K = 8 channels
//     per wgmma.  Row tiles (1x1, and 3x3x3 with N <= 64): a block is 64 consecutive rows, two make a 128-row tile, and
//     3x3x3 halo rows inside it are computed and stored as zeros.  Interior blocks (3x3x3 with N = 128): a block is
//     8 y-lines x 8 z of one x-plane -- halo rows are neither computed nor written.  Blocks are ordered z fastest, then
//     y, then x, and a group of 2 consecutive blocks of one shape is one work item -- 4 (two per warpgroup, twice the
//     MMAs per weight slab and A stage) where B x ceil(blocks / 4) still gives every SM a group (conv_tc_run).
//   * A operand: the activation tensor is [C/4][rows][4] in HBM, i.e. for 4 channels all rows
//     are contiguous at a 16-byte pitch.  That *is* the canonical no-swizzle K-major wgmma
//     layout (core matrix = 8 rows x 16 B = 128 contiguous bytes, SBO between 8-row groups,
//     LBO = distance between channel groups): SBO = 128 B covers 64 consecutive rows, SBO = (r+2) * 16 B covers
//     8 consecutive y-lines of 8 z each.  One contiguous cp.async.bulk per channel group stages a 3x3x3 group's
//     window for one x-plane tap (from row (y0-1, z0-1) of its first block to (y0+8, z0+8) of its last: 10 y-lines x
//     18 z for 2 blocks at r = 16), and every one of the 9 (dy,dz) taps of every block is the SAME shared-memory
//     bytes viewed through a descriptor whose start address is shifted by (dy*(r+2)+dz) rows.  L2->SM traffic per
//     MAC drops 9x versus reloading per tap.
//   * B operand: weights pre-packed [n-tile][chunk][x-plane][tap][C/4][co][4] so one bulk copy
//     brings the 9 taps of a (channel chunk, x-plane) -- or, for interior blocks where that deepens the A ring, one of
//     three copies of 3 taps each (Params::tps); a CTA reuses it for up to tiles_per_item row tiles or 2
//     interior blocks per warpgroup, whose accumulators all stay in registers (<= 128 per thread).
//   * Output contract: rows of [p_begin, p_end) are written (halo rows as zeros), except on interior blocks, which
//     leave the halo rows as they were: every consumer of a 3x3x3 output reads interior rows only.  Each output's
//     accumulation order is the row tiles' (same channel chunks, x-planes, taps, k-steps), and the GroupNorm sums of
//     interior blocks come from k_conv_stats, which re-reads the output and sums it over the row tiles' items with the
//     epilogue's statistics routine (halo_mask, stat_add, stat_flush): results are identical either way.
//   * persistent CTAs (one per SM, 288 threads): warps 0-7 = two consumer warpgroups (wgmma into
//     registers, then the epilogue: +bias -> row mask -> coalesced float4 stores, GroupNorm sum /
//     sum-of-squares per warp in shared memory, one fp64 atomic per channel per shape and item),
//     warp 8 = bulk-copy producer.  4-block groups run 384 threads: warps 8-11 give registers to the consumers (see
//     conv_threads) and warp 8 alone copies.
//   * operand type OP: float (TF32 wgmma, 4 channels per 16-byte group, m64nNk8) or __half (FP16 wgmma, 8 channels per
//     group, m64nNk16; the second 3x3x3 convolution of a PVConv under autocast).  A group is 16 bytes either way and one
//     k-step consumes two of them through the same descriptors, so the tiling record, the rings, the copies and the
//     epilogue are the same bytes; only the MMA instruction reads OP.
#include <algorithm>
#include <type_traits>
#include <cuda_fp16.h>

#include "common.cuh"
#include "model.cuh"
#include "wgmma.cuh"

namespace lion {
namespace tc {

using namespace sm90;

constexpr int CONSUMER_WARPS = 8;                    // two warpgroups: rows 0-63 / 64-127 of every tile
constexpr int THREADS = 32 * CONSUMER_WARPS + 32;    // + warp 8, the producer
// Two interior blocks per warpgroup need two 64-register accumulator sets per thread, more than the 168 registers a
// thread of the 288-thread block gets (each of the SM's 4 register-file quarters holds 3 of its 9 warps).  Those kernels
// run a whole producer warpgroup instead (384 threads, warp 8 copies, warps 9-11 exit) and move registers from it to
// the consumers with setmaxnreg: one producer-warpgroup warp x 96 + two consumer warps x 200 registers per quarter,
// 15,872 of 16,384 (ptxas: no spills; the consumers need about 180).
__host__ __device__ constexpr int conv_threads(int BPW) { return BPW == 2 ? 32 * CONSUMER_WARPS + 128 : THREADS; }
constexpr int PRODUCER_REGS = 96, CONSUMER_REGS = 200;
constexpr int MAX_A_STAGES = 16;   // the A ring is as deep as shared memory allows (Params::a_stages)
constexpr int MAX_B_STAGES = 4;   // the weight ring: 2 slabs, deeper for 3x3x3 where shared memory allows, or 4 3-tap parts (Params::b_stages)
constexpr int OCC_SMEM = 1024;       // bytes of per-item occupancy flags kept in shared memory (r <= 38)
// row tiles per work item: their accumulators (NT / 2 registers per thread each, 64 in all) share one weight slab.  The
// statistics pass (k_conv_stats) rebuilds the row tiles' GroupNorm grouping from it, so it must not change.  Interior
// blocks have their own count per warpgroup (k_conv_tc's BPW, see conv_threads).
__host__ __device__ constexpr int tiles_per_item(int NT) { return NT <= 32 ? 4 : (NT <= 64 ? 2 : 1); }
// fixed shared memory after the A / B rings: bias, per-warp GroupNorm partials, the pooled epilogue's exchange (1x1 only),
// barriers + flags, occupancy flags.  What the kernel does not use is left to the A ring.
constexpr int SMEM_BIAS = 128 * 4, SMEM_BARS = 64 * 8 + 128;
__host__ __device__ constexpr int smem_stat(int NT) { return CONSUMER_WARPS * 2 * NT * 4; }
__host__ __device__ constexpr int smem_pool(int NT, int TPG) { return TPG == 1 ? CONSUMER_WARPS * 2 * NT * 4 : 0; }
__host__ __device__ constexpr int smem_fixed(int NT, int TPG) {
  return SMEM_BIAS + smem_stat(NT) + smem_pool(NT, TPG) + SMEM_BARS + OCC_SMEM;
}

struct Params {
  const float4* in; const float* w; const float* bias; float4* out; double* ssum; double* ssq;
  int Gin, Gout_store, cout_pad;
  int rows;              // rows per (b, group)
  int p_begin, p_end;    // 1x1: the rows computed
  int ntile;             // tiles per shape: 1x1 128-row tiles, 3x3x3 block groups (see k_conv_tc)
  int ntg, tpg;          // tap groups (x planes) and taps per group: (3,9) or (1,1)
  int tg_off[3];         // row offset of each tap group (dx * rp^2)
  int tap_off[9];        // row offset of each tap inside a group (dy*rp + dz)
  // 3x3x3 block geometry: r, rp = r+2, z / y blocks per x plane (ceil(r/8)), blocks per shape, blocks per group
  int r, rp, nzb, npl, nblk, ib;
  int halo;              // 3x3x3 row tiles: rp+1 rows before and after the tile in the operand slab, else 0
  int KG, nchunk;        // channel groups per chunk, chunks
  int NT;                // output channels per CTA (wgmma N)
  int G;                 // tiles per work item (1 for 3x3x3: a block group is one item)
  int B;                 // shapes
  int a_stage_bytes, b_stage_bytes, stage_rows;
  int a_stages;          // depth of the A ring
  int b_stages;          // depth of the weight ring
  int tps;               // taps per weight stage: tpg (whole slabs), or 3 (3x3x3 slabs streamed in 3-tap parts)
  const unsigned char* occ;   // 64-row occupancy flags of the input (sparse first conv of a PVConv) or null
  int occ_stride;
  // 3x3x3 row tiles: one byte per 64-row block of [p_begin, p_end) per shape ([B][cls_stride], block k = rows p_begin +
  // 64 k ..), set where every operand of every interior row is a per-channel constant or a halo zero (k_conv2_flags), or
  // null.  A flagged block's outputs are its rows' border-class values, cls [B][cout_pad / 4][5^3]: the same convolution
  // of a 3x3x3 grid of those constants (row ((cx+1) * 5 + cy+1) * 5 + cz+1 for the low / interior / high class 0 / 1 / 2
  // of x, y and z).  Its MMAs and copies are skipped; its rows are stored only when cls_store.
  const unsigned char* cls_flag;
  int cls_stride;
  const float4* cls;
  int cls_store;
  // pooled 1x1 (last layer of a set-abstraction MLP): instead of the [rows][C] result, write per 32 consecutive rows (the
  // neighbours of one centre) the per-channel minimum and maximum, pool_mm[b][C/4][rows/32][2][4].  AdaGN's affine is
  // monotonic and Swish is quasi-convex (one minimum), so max_i swish(s*x_i + t) = max(swish(s*min + t), swish(s*max + t)):
  // the consumer needs 2 of the 32 values.
  float* pool_mm;
  int sched;             // work distribution: 0 contiguous range per CTA, 1 interleaved items (see k_conv_tc)
};

// 3x3x3: first row of block k of a shape (8 y-lines x 8 z of one x plane; blocks ordered z fastest, then y, then x)
__host__ __device__ __forceinline__ int block_row(int k, int rp, int nzb, int npl) {
  const int x = k / npl, rem = k - x * npl, yb = rem / nzb, zb = rem - yb * nzb;
  return ((x + 1) * rp + 1 + 8 * yb) * rp + 1 + 8 * zb;
}

// all wgmmas of NB 64-row blocks (operands at a_addr[0 .. NB-1]) for TPG consecutive taps of one (channel chunk, tap
// group) of this warpgroup (weights of the first at b_addr, row offsets tap_off[0 .. TPG-1]): TPG taps x KG/2 k-steps,
// the blocks interleaved per k-step (each accumulator set d[k] still takes its taps and k-steps in order; the blocks
// share the weight descriptors).  a_sbo is the distance between a block's 8-row groups: 128 B for 64 consecutive rows,
// (r+2) * 16 B for 8 y-lines x 8 z.
template <int KG, int TPG, int NT, int NB = 1, typename OP = float>
__device__ __forceinline__ void issue_stage(float (*d)[NT / 2], const uint32_t* a_addr, uint32_t b_addr, uint32_t a_pitch,
                                            uint32_t a_sbo, const int* tap_off) {
  const uint64_t b0 = make_desc(b_addr, NT * 16, 128);
  uint64_t a0[NB];
#pragma unroll
  for (int k = 0; k < NB; ++k) a0[k] = make_desc(a_addr[k], a_pitch, a_sbo);
#pragma unroll
  for (int t = 0; t < TPG; ++t) {
    const uint64_t toff = (uint64_t)(int64_t)(TPG == 1 ? 0 : tap_off[t]);      // descriptor address unit = 16 B = 1 row
#pragma unroll
    for (int ks = 0; ks < KG / 2; ++ks)
#pragma unroll
      for (int k = 0; k < NB; ++k) {
        const uint64_t a = a0[k] + toff + (uint64_t)((ks * 2 * a_pitch) >> 4), b = b0 + (uint64_t)(((t * KG + ks * 2) * NT * 16) >> 4);
        if constexpr (std::is_same<OP, __half>::value) wgmma_f16<NT>(d[k], a, b, 1);
        else wgmma_tf32<NT>(d[k], a, b, 1);
      }
  }
}


struct Items {
  long long u, u_end; int ntile_total, B, G;
  int mode, m, q, n_p, n_q, c_i, i, big, k;   // sched 1: [u, u_end) is the rest of the current item (cut at n-tile boundaries)
  // next item: n-tile nt, first tile v0 in the n-tile's flat (shape, row tile) space, ntile tiles.  An item may run
  // across a shape boundary -- its tiles share the weight slabs whatever shape they belong to -- but not across n-tiles.
  __device__ __forceinline__ bool next(int& nt, long long& v0, int& ntile) {
    const long long per_nt = (long long)B * ntile_total;
    if (mode) {
      while (u >= u_end) {
        if (k >= m) return false;
        const int a0 = q * k / m, a1 = q * (k + 1) / m, b0 = (q + 1) * k / m, b1 = (q + 1) * (k + 1) / m;
        u = (long long)n_q * a0 + (long long)n_p * b0 + (long long)(i - c_i) * (a1 - a0) + (long long)c_i * (b1 - b0);
        u_end = u + (big ? b1 - b0 : a1 - a0);
        ++k;
      }
      nt = (int)(u / per_nt);
      v0 = u - (long long)nt * per_nt;
      const long long lim = (long long)(nt + 1) * per_nt;
      const long long e = u_end < lim ? u_end : lim;
      ntile = (int)(e - u);          // <= ceil((q + 1) / m) <= G
      u = e;
      return true;
    }
    if (u >= u_end) return false;
    nt = (int)(u / per_nt);
    v0 = u - (long long)nt * per_nt;
    long long run = per_nt - v0;
    if (u_end - u < run) run = u_end - u;
    const long long k2 = (run + G - 1) / G;
    ntile = (int)((run + k2 - 1) / k2);
    u += ntile;
    return true;
  }
};
// the items of CTA blockIdx.x out of gridDim.x over U = n-tiles x shapes x tiles (see k_conv_tc: work distribution)
__device__ __forceinline__ Items make_items(long long U, int ntile_total, int B, int G, int sched) {
  const long long u_begin = U * blockIdx.x / gridDim.x, u_end = U * (blockIdx.x + 1) / gridDim.x;
  Items it{u_begin, u_end, ntile_total, B, G, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  if (sched) {
    const int grid = (int)gridDim.x, q = (int)(U / grid), n_p = (int)(U - (long long)q * grid);
    const int tmax = q + (n_p ? 1 : 0);
    it.mode = 1; it.u = 0; it.u_end = 0;
    it.m = (tmax + G - 1) / G; it.q = q; it.n_p = n_p; it.n_q = grid - n_p;
    it.i = (int)blockIdx.x; it.c_i = (int)(u_begin - (long long)q * blockIdx.x);
    it.big = (int)(u_end - u_begin) > q; it.k = 0;
  }
  return it;
}

// border class of coordinate v (1 .. r) of a 3x3x3 row tile: 0 low, 1 interior, 2 high (Params::cls)
__device__ __forceinline__ int cls_of(int v, int r) { return v <= 1 ? 0 : (v >= r ? 2 : 1); }

// GroupNorm statistics in the row tiles' grouping, shared by k_conv_tc's epilogue and k_conv_stats so that both sum
// alike: per fragment a shuffle tree over the warp's 8 row pairs, per-warp fp32 partials in s_stat [8 consumer warps]
// [sum, sum of squares][NT], and per (shape, item) a fixed-order sum over the warps with one fp64 atomic per channel.
//
// 3x3x3 row tiles: rows p_lo and p_lo + 8 of a fragment that are y / z halo rows of their x plane count as zeros.
__device__ __forceinline__ void halo_mask(int p_lo, int rp, bool& ok_lo, bool& ok_hi) {
  const int p_hi = p_lo + 8;
  const int z0 = p_lo % rp, y0 = (p_lo / rp) % rp, z1 = p_hi % rp, y1 = (p_hi / rp) % rp;
  ok_lo = ok_lo && z0 >= 1 && z0 <= rp - 2 && y0 >= 1 && y0 <= rp - 2;
  ok_hi = ok_hi && z1 >= 1 && z1 <= rp - 2 && y1 >= 1 && y1 <= rp - 2;
}
// adds one fragment -- channels col, col + 1 of rows p_lo (x0, x1) and p_lo + 8 (x2, x3) -- to consumer warp cw's partials
template <int NT>
__device__ __forceinline__ void stat_add(float* s_stat, int cw, int lane, int col, float x0, float x1, float x2, float x3) {
  const float s0 = red8<0>(x0 + x2), s1 = red8<0>(x1 + x3);
  const float q0 = red8<0>(fmaf(x0, x0, x2 * x2)), q1 = red8<0>(fmaf(x1, x1, x3 * x3));
  if (lane < 4) {
    float* st = s_stat + (cw * 2) * NT + col;
    st[0] += s0; st[1] += s1; st[NT] += q0; st[NT + 1] += q1;
  }
}
// moves the partials of shape b, channels n0 .. n0 + NT - 1 into ssum / ssq and zeroes them.  Named barrier 1 over the
// 256 consumer threads (k_conv_tc's producer warp never gets here): every one of them must call it.
template <int NT>
__device__ __forceinline__ void stat_flush(const Params& P, float* s_stat, int et, int b, int n0) {
  asm volatile("bar.sync 1, 256;" ::: "memory");
  if (et < NT) {
    float s = 0.f, qq = 0.f;
#pragma unroll
    for (int w = 0; w < CONSUMER_WARPS; ++w) {
      s += s_stat[(w * 2 + 0) * NT + et]; qq += s_stat[(w * 2 + 1) * NT + et];
      s_stat[(w * 2 + 0) * NT + et] = 0.0f; s_stat[(w * 2 + 1) * NT + et] = 0.0f;
    }
    atomicAdd(P.ssum + (size_t)b * P.cout_pad + n0 + et, (double)s);
    atomicAdd(P.ssq + (size_t)b * P.cout_pad + n0 + et, (double)qq);
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");
}

// BLK: 3x3x3 on interior 8 x 8 blocks (TPG == 9), BPW of them per warpgroup and group (P.ib = 2 * BPW); otherwise
// 128-row tiles.  TPS: taps per weight stage (= P.tps), TPG or 3; a commit group's wgmmas are one static chain.
// OP: operand type of the MMAs (float = TF32, __half = FP16), see the header.
template <int KG, int TPG, int NT, bool BLK, int BPW = 1, int TPS = TPG, typename OP = float>
__global__ void __launch_bounds__(conv_threads(BPW), 1) k_conv_tc(Params P) {
  constexpr int GT = BLK ? BPW : tiles_per_item(NT);   // accumulator sets per thread
  constexpr int NTHR = conv_threads(BPW);
  constexpr bool SETREG = NTHR > THREADS;              // registers moved from the producer warpgroup to the consumers
  constexpr int NACC = NT / 2;                  // accumulator registers per thread and tile
  constexpr int NPARTS = TPG / TPS;             // weight stages per (channel chunk, x-plane) slab
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sA = smem;
  const int A_STAGES = P.a_stages;
  uint8_t* sB = sA + (size_t)A_STAGES * P.a_stage_bytes;
  const int B_STAGES = P.b_stages;
  float* s_bias = (float*)(sB + (size_t)B_STAGES * P.b_stage_bytes);
  float* s_stat = s_bias + 128;                 // [8 consumer warps][2][NT]: running GroupNorm partials of the current shape
  float* s_pool = s_stat + CONSUMER_WARPS * 2 * NT;    // [8 consumer warps][2][NT]: pooled-epilogue exchange (TPG == 1)
  uint64_t* bars = (uint64_t*)((uint8_t*)s_stat + smem_stat(NT) + smem_pool(NT, TPG));
  volatile uint32_t* s_skip = (volatile uint32_t*)(bars + 64);   // [MAX_A_STAGES] stage holds no data (all-zero input slab)
  uint8_t* s_occ = (uint8_t*)(bars + 64) + 128;  // [OCC_SMEM] this item's 64-row occupancy flags (sparse first convolution)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  const uint32_t bar_full_a = smem_u32(bars), bar_empty_a = smem_u32(bars + MAX_A_STAGES);
  const uint32_t bar_full_b = smem_u32(bars + 2 * MAX_A_STAGES), bar_empty_b = smem_u32(bars + 2 * MAX_A_STAGES + MAX_B_STAGES);

  // zero the A stages once: channel-group slots that a partial chunk does not load must hold
  // finite values (their weights are zero)
  if (P.Gin % KG != 0)
    for (int i = tid; i < A_STAGES * P.a_stage_bytes / 16; i += NTHR) ((float4*)sA)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = tid; i < CONSUMER_WARPS * 2 * NT; i += NTHR) s_stat[i] = 0.0f;
  if (tid == 0) {
    // a stage is released by every consumer warp once its wgmmas have read it
    for (int i = 0; i < A_STAGES; ++i) { mbar_init(bar_full_a + 8 * i, 1); mbar_init(bar_empty_a + 8 * i, CONSUMER_WARPS); }
    for (int i = 0; i < B_STAGES; ++i) { mbar_init(bar_full_b + 8 * i, 1); mbar_init(bar_empty_b + 8 * i, CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy zero fill -> async proxy readers
  __syncthreads();

  // Work distribution.  The (n-tile, shape, tile) space is flattened (tile fastest) and cut into work items = up to G
  // consecutive tiles sharing the weight slabs (they may belong to two shapes, never to two n-tiles).  A 1x1 tile is 128
  // consecutive rows; on interior blocks a tile is one group of ib blocks, and G = 1 (the group already shares the weight slabs and has
  // one operand window, so it never spans two shapes).  3x3x3 tiles are ordered x-major like the rows.  Every CTA gets
  // the same number of tiles (+-1): fixed G-tile items dealt round-robin would leave some CTAs half again as many tiles as
  // others, and the kernel runs at the pace of the busiest.
  //   sched 0: one contiguous range per CTA, cut into evenly sized items (9 tiles -> 3+3+3, not 4+4+1).  Balanced, but at
  //            r = 32 the CTAs then stream as many distant windows of a 268 MB input at once: the 3 x-plane sweeps of a tile
  //            (9 tiles apart) miss the L2 and the input is read from DRAM up to three times.
  //   sched 1: the same tiles per CTA T_i (= the contiguous range's size) and the same number of items m = ceil(max T / G), but
  //            dealt in m ROUNDS: round k is one contiguous stretch of the tile space, cut into one item per CTA (CTA i's item
  //            has floor(T_i (k+1) / m) - floor(T_i k / m) tiles).  At any moment the CTAs work on ~grid ADJACENT items
  //            (a few shapes), so a tile's x-plane neighbours are in flight in a neighbouring CTA and hit the L2.
  //            With T_i in {q, q+1} every offset has a closed form: A_k = floor(q k / m), B_k = floor((q+1) k / m),
  //            c_i = CTAs before i that own q+1 tiles;  start(i, k) = n_q A_k + n_p B_k + (i - c_i)(A_k+1 - A_k) + c_i (B_k+1 - B_k).
  const int ntile_total = P.ntile;
  const int n_nt = P.cout_pad / P.NT;
  const long long U = (long long)n_nt * P.B * ntile_total;
  const Items items0 = make_items(U, ntile_total, P.B, P.G, P.sched);

  if (warp >= CONSUMER_WARPS) {
    // ===================== producer (whole warp; lane kg issues the copy of channel group kg) ====
    if constexpr (SETREG) {
      regs_dec<PRODUCER_REGS>();
      if (warp > CONSUMER_WARPS) return;
    }
    uint32_t sa = 0, pa = 0, sb = 0, pb = 0;          // ring positions and phase bits
    const uint32_t bytes = (uint32_t)P.stage_rows * 16u;
    const uint32_t sA_addr = smem_u32(sA), sB_addr = smem_u32(sB);
    Items items = items0;
    int nt, ntile;
    long long v0;
    int occ_shape = -1;                                // shape whose occupancy flags s_occ holds
    const int slab_floats = P.tpg * KG * NT * 4;       // one (chunk, x-plane) of the packed weights: tpg taps
    auto copy_weights = [&](const float* src) {        // the next weight stage: tps taps from src
      mbar_wait<SETREG>(bar_empty_b + 8 * sb, pb ^ 1);
      if (lane == 0) {
        mbar_expect_tx(bar_full_b + 8 * sb, P.b_stage_bytes);
        bulk_g2s(sB_addr + sb * (uint32_t)P.b_stage_bytes, src, P.b_stage_bytes, bar_full_b + 8 * sb);
      }
      if (++sb == B_STAGES) { sb = 0; pb ^= 1; }
    };
    while (items.next(nt, v0, ntile)) {
      const float* wsrc = P.w + (size_t)nt * P.nchunk * P.ntg * slab_floats;
      // lane l keeps (shape, row tile) of the item's tile l: one division per item, a shuffle per stage
      int my_b = 0, my_t = 0;
      if (lane < ntile) { const int vl = (int)v0 + lane; my_b = vl / ntile_total; my_t = vl - my_b * ntile_total; }
      // tiles with an operand to copy: all but those whose two 64-row blocks are both class-valued (the consumers
      // compute the same set and skip the same ring slots)
      unsigned live = (1u << ntile) - 1u;
      if (!BLK && P.cls_flag) {
        const unsigned char* fl = P.cls_flag + (size_t)my_b * P.cls_stride + 2 * my_t;
        live = __ballot_sync(0xffffffffu, lane < ntile && !(__ldg(fl) && __ldg(fl + 1)));
      }
      if (!live) continue;                             // every output of the item is a class value: no weights either
      for (int cc = 0; cc < P.nchunk; ++cc) {
        const int kg_real = min(KG, P.Gin - cc * KG);
        const size_t grp_lane = (size_t)(cc * KG + (lane < kg_real ? lane : 0));
        for (int tg = 0; tg < P.ntg; ++tg) {
          // the last sweep of an item is never skipped: every accumulator then receives at
          // least one (zero-initialising) MMA per item and needs no "was it touched" bookkeeping
          const bool may_skip = P.occ && !(cc == P.nchunk - 1 && tg == P.ntg - 1);
          // the slab's first weight stage, its tiles' A stages, then the slab's other parts: the order in which the
          // consumers wait for them
          const float* slab = wsrc + (size_t)(cc * P.ntg + tg) * slab_floats;
          copy_weights(slab);
          for (int j = 0; j < ntile; ++j) {
            if (!((live >> j) & 1u)) continue;
            const int bj = __shfl_sync(0xffffffffu, my_b, j), tj = __shfl_sync(0xffffffffu, my_t, j);
            // row tiles: the tile's 128 rows (3x3x3: plus rp+1 halo rows on each side, shifted to x-plane tg).  Interior
            // blocks: the window of block group tj under tap group tg, from one row before
            // its first block's (-1, -1) neighbour; the last group's window is cut at the end of the shape's rows
            long long row0;
            uint32_t cnt = (uint32_t)P.stage_rows;
            if (!BLK) {
              row0 = (long long)P.p_begin + (long long)tj * 128 - P.halo + P.tg_off[tg];
            } else {
              row0 = (long long)block_row(tj * P.ib, P.rp, P.nzb, P.npl) - P.rp - 1 + P.tg_off[tg];
              if (row0 + cnt > (long long)P.rows) cnt = (uint32_t)(P.rows - row0);
            }
            const float4* in_lane = P.in + ((size_t)bj * P.Gin + grp_lane) * P.rows;
            mbar_wait<SETREG>(bar_empty_a + 8 * sa, pa ^ 1);
            bool empty = false;
            if (may_skip) {
              // sparse input: the shape's occupancy flags (<= 1 KB) live in shared memory -- a broadcast LDS per
              // check instead of dependent global loads on the producer's critical path
              const unsigned char* occ_b = P.occ + (size_t)bj * P.occ_stride;
              if (P.occ_stride <= OCC_SMEM) {
                if (occ_shape != bj) {
                  __syncwarp();
                  for (int k = lane; k < P.occ_stride; k += 32) s_occ[k] = __ldg(occ_b + k);
                  __syncwarp();
                  occ_shape = bj;
                }
                occ_b = s_occ;
              }
              long long lo = row0 < 0 ? 0 : row0, hi = row0 + cnt - 1;
              if (hi > P.rows - 1) hi = P.rows - 1;
              unsigned any = 0;
              for (int k = (int)(lo >> 6); k <= (int)(hi >> 6); ++k) any |= occ_b[k];
              empty = (any == 0);
            }
            const uint32_t full = bar_full_a + 8 * sa;
            if (lane == 0) {
              s_skip[sa] = empty ? 1u : 0u;
              if (empty) asm volatile("mbarrier.arrive.release.cta.shared::cta.b64 _, [%0];" ::"r"(full) : "memory");
              else mbar_expect_tx(full, cnt * 16u * kg_real);
            }
            __syncwarp();
            if (!empty && lane < kg_real)
              bulk_g2s(sA_addr + sa * (uint32_t)P.a_stage_bytes + lane * bytes, in_lane + row0, cnt * 16u, full);
            if (++sa == (uint32_t)A_STAGES) { sa = 0; pa ^= 1; }
          }
          for (int s = 1; s < NPARTS; ++s) copy_weights(slab + (size_t)s * (P.b_stage_bytes / 4));
        }
      }
    }
  } else {
    // ===================== consumers ===========
    // row tiles: warpgroup wg computes rows 64 wg .. 64 wg + 63 of every tile.  Interior blocks: blocks wg, wg + 2, ...
    if constexpr (SETREG) regs_inc<CONSUMER_REGS>();
    const int cw = warp, wg = cw >> 2, wq = cw & 3;
    const int et = tid;                                  // 0..255
    const uint32_t a_pitch = (uint32_t)P.stage_rows * 16u;
    const uint32_t a_sbo = BLK ? (uint32_t)P.rp * 16u : 128u;
    const uint32_t a_ring = smem_u32(sA) + (BLK ? 0u : (uint32_t)(P.halo + 64 * wg) * 16u);
    const uint32_t b_ring = smem_u32(sB);
    const int r_lo = 64 * wg + 16 * wq + (lane >> 2);   // 1x1: this thread's rows of a tile: r_lo and r_lo + 8,
    const int c_lo = 2 * (lane & 3);                     // its columns: 8 i + c_lo and 8 i + c_lo + 1
    const bool odd = (lane & 1) != 0;
    float acc[GT][NACC];
    uint32_t sa = 0, pa = 0, sb = 0, pb = 0;
    Items items = items0;
    int nt, ntile;
    long long v0;
    auto release = [&](int& s, uint32_t bar0) {
      if (s >= 0) { if (lane == 0) mbar_arrive(bar0 + 8 * s); s = -1; }
    };
    while (items.next(nt, v0, ntile)) {
#pragma unroll
      for (int j = 0; j < GT; ++j)
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[j][i] = 0.0f;
      // 3x3x3: this warpgroup's nbw blocks of the group (first block g_f) and their offsets in the window.  All GT
      // blocks are issued (a wgmma under a branch would serialise them all): a block past the shape's last one reads the
      // group's first block, and its accumulators are not stored.
      int g_f = 0, nbw = 0;
      uint32_t boff[GT];
      if (BLK) {
        const int g_b = (int)(v0 / ntile_total);
        g_f = (int)(v0 - (long long)g_b * ntile_total) * P.ib;
        const int nb = min(P.ib, P.nblk - g_f);
        nbw = (nb - wg + 1) / 2;
        const int s_f = block_row(g_f, P.rp, P.nzb, P.npl);
#pragma unroll
        for (int j = 0; j < GT; ++j) {
          const int k = 2 * j + wg < nb ? g_f + 2 * j + wg : g_f;
          boff[j] = (uint32_t)(block_row(k, P.rp, P.nzb, P.npl) - s_f + P.rp + 1) * 16u;
        }
      }
      // A stage (and weight stage) handed back one commit group late (wait_group 1): the tensor cores work on the
      // next group while this warp checks that the previous one has been read.  A slab streamed in parts is one
      // commit group per (part, tile): every accumulator still takes taps 0-8 in order, and a tile's A stage is held
      // until the group of its last part has completed.
      int pend_a = -1, pend_b = -1;
      bool skip[BLK ? 1 : GT];
      // row tiles with class-valued blocks (Params::cls_flag): `live` tiles have an A stage (the producer's set), `mine`
      // those whose block of this warpgroup is computed
      unsigned live = (1u << ntile) - 1u, mine = ~0u;
      if (!BLK && P.cls_flag) {
        live = 0u; mine = 0u;
#pragma unroll
        for (int j = 0; j < GT; ++j) {
          if (j < ntile) {
            const long long vj = v0 + j;
            const int bj = (int)(vj / ntile_total), tj = (int)(vj - (long long)bj * ntile_total);
            const unsigned char* fl = P.cls_flag + (size_t)bj * P.cls_stride + 2 * tj;
            const bool f0 = __ldg(fl) != 0, f1 = __ldg(fl + 1) != 0;
            if (!(f0 && f1)) live |= 1u << j;
            if (!(wg ? f1 : f0)) mine |= 1u << j;
          }
        }
      }
      for (int cc = 0; cc < (live ? P.nchunk : 0); ++cc) {
        for (int tg = 0; tg < P.ntg; ++tg) {
          const uint32_t sa0 = sa, pa0 = pa;             // A stage of the slab's first tile
#pragma unroll
          for (int s = 0; s < NPARTS; ++s) {
            mbar_wait<SETREG>(bar_full_b + 8 * sb, pb);
            const uint32_t b_addr = b_ring + sb * (uint32_t)P.b_stage_bytes;
            const int* toff = P.tap_off + s * TPS;
            bool issued = false;
            sa = sa0; pa = pa0;
#pragma unroll
            for (int j = 0; j < (BLK ? 1 : GT); ++j) {
              if ((live >> j) & 1u) {
                if (s == 0) {
                  mbar_wait<SETREG>(bar_full_a + 8 * sa, pa);
                  // all-zero input slab (nothing to accumulate), or this warpgroup's block is class-valued
                  skip[j] = s_skip[sa] != 0 || !((mine >> j) & 1u);
                  if (skip[j]) { int st = (int)sa; release(st, bar_empty_a); }
                }
                if (!skip[j]) {
                  const uint32_t a_addr = a_ring + sa * (uint32_t)P.a_stage_bytes;
                  wg_fence();
                  if (!BLK) {
                    issue_stage<KG, TPS, NT, 1, OP>(&acc[j], &a_addr, b_addr, a_pitch, a_sbo, toff);
                  } else {
                    uint32_t a_blk[GT];
#pragma unroll
                    for (int k = 0; k < GT; ++k) a_blk[k] = a_addr + boff[k];
                    issue_stage<KG, TPS, NT, GT, OP>(acc, a_blk, b_addr, a_pitch, a_sbo, toff);
                  }
                  wg_commit();
                  wg_wait<1>();
                  release(pend_a, bar_empty_a);
                  release(pend_b, bar_empty_b);
                  if (s == NPARTS - 1) pend_a = (int)sa;  // the tile's last group: its A stage goes back after it
                  issued = true;
                }
                if (++sa == (uint32_t)A_STAGES) { sa = 0; pa ^= 1; }
              }
            }
            if (pend_b >= 0) {                           // no group issued on this stage: retire the older one
              wg_wait<0>();
              release(pend_a, bar_empty_a);
              release(pend_b, bar_empty_b);
            }
            if (issued) pend_b = (int)sb;                // the group in flight still reads this weight stage
            else { int st = (int)sb; release(st, bar_empty_b); }
            if ((live & ~mine) && pend_b >= 0) {          // see conv_tc_run: class-valued blocks and the A ring
              wg_wait<0>();
              release(pend_a, bar_empty_a);
              release(pend_b, bar_empty_b);
            }
            if (++sb == B_STAGES) { sb = 0; pb ^= 1; }
          }
        }
      }
      wg_wait<0>();
      release(pend_a, bar_empty_a);
      release(pend_b, bar_empty_b);
#pragma unroll
      for (int j = 0; j < GT; ++j) fence_regs<NACC>(acc[j]);

      // ---- epilogue, straight from the accumulator registers
      const int n0 = nt * NT;
      asm volatile("bar.sync 1, 256;" ::: "memory");    // previous item's s_bias readers are done
      if (et < NT) s_bias[et] = P.bias ? P.bias[n0 + et] : 0.0f;
      asm volatile("bar.sync 1, 256;" ::: "memory");
      // GroupNorm statistics are per shape: flushed whenever the item moves on to the next shape, and at its end
      int b = (int)(v0 / ntile_total);
#pragma unroll
      for (int j = 0; j < GT; ++j) {
        if (j < (BLK ? nbw : ntile)) {
          int tj = 0, p_lo, p_hi;
          bool ok_lo, ok_hi;
          bool in_lo, in_hi;
          if (!BLK) {
            const long long vj = v0 + j;
            const int bj = (int)(vj / ntile_total);
            tj = (int)(vj - (long long)bj * ntile_total);
            if (bj != b) { if (P.ssum) stat_flush<NT>(P, s_stat, et, b, n0); b = bj; }
            p_lo = P.p_begin + tj * 128 + r_lo; p_hi = p_lo + 8;
            in_lo = p_lo < P.p_end; in_hi = p_hi < P.p_end;
            ok_lo = in_lo; ok_hi = in_hi;
            if (TPG != 1) halo_mask(p_lo, P.rp, ok_lo, ok_hi);   // halo rows are stored as zeros
            if (!((mine >> j) & 1u)) {
              // class-valued block: the accumulators take the border-class values of their rows (the bias included)
              // and the statistics below sum them as they would the computed ones
              const float4* cb = P.cls + (size_t)b * (P.cout_pad / 4) * 125 + n0 / 4;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int p = h ? p_hi : p_lo, x = p / (P.rp * P.rp), y = (p / P.rp) % P.rp, z = p % P.rp;
                const int row = ((cls_of(x, P.r) + 1) * 5 + cls_of(y, P.r) + 1) * 5 + cls_of(z, P.r) + 1;
                // channels n0 + 8 i + c_lo, + 1: group n0 / 4 + 2 i + (lane & 3) / 2, floats 2 (lane & 1), + 1
                const float* src = reinterpret_cast<const float*>(cb + ((lane & 3) >> 1) * 125 + row) + 2 * (lane & 1);
#pragma unroll
                for (int i = 0; i < NT / 8; ++i) {
                  const float2 v = __ldg(reinterpret_cast<const float2*>(src + (size_t)2 * 125 * 4 * i));
                  acc[j][4 * i + 2 * h] = v.x; acc[j][4 * i + 2 * h + 1] = v.y;
                }
              }
            }
          } else {
            // fragment row i of block k is voxel (y0 + i / 8, z0 + i % 8): this thread's rows are y-lines y0 + 2 wq
            // and y0 + 2 wq + 1 at z0 + lane / 4.  Rows past r (a last block of an r that is not a multiple of 8) are
            // neither stored nor counted.
            const int k = g_f + 2 * j + wg, x = k / P.npl, rem = k - x * P.npl, yb = rem / P.nzb, zb = rem - yb * P.nzb;
            const int y = 1 + 8 * yb + 2 * wq, z = 1 + 8 * zb + (lane >> 2);
            p_lo = ((x + 1) * P.rp + y) * P.rp + z; p_hi = p_lo + P.rp;
            ok_lo = y <= P.r && z <= P.r; ok_hi = y + 1 <= P.r && z <= P.r;
            in_lo = ok_lo; in_hi = ok_hi;
          }
          const bool cmp = (mine >> j) & 1u, st = cmp || P.cls_store;   // computed block / rows stored
#pragma unroll
          for (int i = 0; i < NT / 8; ++i) {
            const int col = 8 * i + c_lo;
            float x0 = acc[j][4 * i + 0], x1 = acc[j][4 * i + 1], x2 = acc[j][4 * i + 2], x3 = acc[j][4 * i + 3];
            if (cmp) { x0 += s_bias[col]; x1 += s_bias[col + 1]; x2 += s_bias[col]; x3 += s_bias[col + 1]; }
            x0 = ok_lo ? x0 : 0.0f; x1 = ok_lo ? x1 : 0.0f; x2 = ok_hi ? x2 : 0.0f; x3 = ok_hi ? x3 : 0.0f;
            if (P.ssum) stat_add<NT>(s_stat, cw, lane, col, x0, x1, x2, x3);
            if (TPG == 1 && P.pool_mm) {                 // all rows valid (rows % 128 == 0)
              const float mn0 = red8<1>(fminf(x0, x2)), mn1 = red8<1>(fminf(x1, x3));
              const float mx0 = red8<2>(fmaxf(x0, x2)), mx1 = red8<2>(fmaxf(x1, x3));
              if (lane < 4) {
                float* sp = s_pool + (cw * 2) * NT + col;
                sp[0] = mn0; sp[1] = mn1; sp[NT] = mx0; sp[NT + 1] = mx1;
              }
            } else {
              // lanes 2k, 2k+1 hold channels 0-1 / 2-3 of a 4-channel group: swap halves so that each stores one float4
              const float y0 = __shfl_xor_sync(0xffffffffu, odd ? x0 : x2, 1);
              const float y1 = __shfl_xor_sync(0xffffffffu, odd ? x1 : x3, 1);
              const int g = (n0 + 8 * i + (lane & 2) * 2) >> 2;
              if (g < P.Gout_store) {
                float4* o = P.out + ((size_t)b * P.Gout_store + g) * P.rows;
                if (!odd && in_lo && st) o[p_lo] = make_float4(x0, x1, y0, y1);
                if (odd && in_hi && st) o[p_hi] = make_float4(y0, y1, x2, x3);
              }
            }
          }
          if (TPG == 1 && P.pool_mm) {
            // a centre's 32 rows are the fragments of warps 2k and 2k+1 of the warpgroup
            const int bar_id = 2 + wg;
            asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
            const long long ncent = (long long)P.rows / 32;
            for (int e = et - 128 * wg; e < 2 * NT; e += 128) {
              const int k = e / NT, c = e - k * NT;
              const float* s0 = s_pool + ((4 * wg + 2 * k) * 2) * NT + c;
              const float* s1 = s0 + 2 * NT;
              const float mn = fminf(s0[0], s1[0]), mx = fmaxf(s0[NT], s1[NT]);
              const long long centre = (long long)(P.p_begin + tj * 128 + 64 * wg + 32 * k) >> 5;
              const int ch = n0 + c;
              float* dst = P.pool_mm + ((((size_t)b * (P.cout_pad / 4) + (ch >> 2)) * ncent + centre) * 2) * 4 + (ch & 3);
              dst[0] = mn; dst[4] = mx;
            }
            asm volatile("bar.sync %0, 128;" ::"r"(bar_id) : "memory");
          }
        }
      }
      if (P.ssum) stat_flush<NT>(P, s_stat, et, b, n0);
    }
  }
}

// GroupNorm statistics of a 3x3x3 output computed on interior blocks, read back from the stored output and summed by
// the row tiles' items and warps through the epilogue's own routine (halo_mask, stat_add, stat_flush).  The fp32
// partials of a different grouping would round differently, and the denoising loop amplifies a one-ulp change of an
// AdaGN scale over its 1000 steps; this pass keeps the statistics -- and so every output -- identical to the row tiles'.
template <int NT>
__global__ void __launch_bounds__(256) k_conv_stats(Params P) {
  constexpr int GT = tiles_per_item(NT);
  __shared__ float s_stat[CONSUMER_WARPS * 2 * NT];
  const int tid = threadIdx.x, cw = tid >> 5, lane = tid & 31, wg = cw >> 2, wq = cw & 3, et = tid;
  for (int i = tid; i < CONSUMER_WARPS * 2 * NT; i += 256) s_stat[i] = 0.0f;
  __syncthreads();
  const int r_lo = 64 * wg + 16 * wq + (lane >> 2), c_lo = 2 * (lane & 3);
  const int ntile_total = P.ntile;
  const long long U = (long long)(P.cout_pad / NT) * P.B * ntile_total;
  Items items = make_items(U, ntile_total, P.B, P.G, P.sched);
  int nt, ntile;
  long long v0;
  while (items.next(nt, v0, ntile)) {
    const int n0 = nt * NT;
    int b = (int)(v0 / ntile_total);
#pragma unroll
    for (int j = 0; j < GT; ++j) {
      if (j < ntile) {
        const long long vj = v0 + j;
        const int bj = (int)(vj / ntile_total), tj = (int)(vj - (long long)bj * ntile_total);
        if (bj != b) { stat_flush<NT>(P, s_stat, et, b, n0); b = bj; }
        const int p_lo = P.p_begin + tj * 128 + r_lo, p_hi = p_lo + 8;
        bool ok_lo = p_lo < P.p_end, ok_hi = p_hi < P.p_end;
        halo_mask(p_lo, P.rp, ok_lo, ok_hi);
        // all of the tile's loads are issued before the first sum: the shuffles and shared-memory adds of stat_add would
        // otherwise hold each load back behind the previous one's, one memory latency per channel group
        float2 lo[NT / 8], hi[NT / 8];
#pragma unroll
        for (int i = 0; i < NT / 8; ++i) {
          const int ch = n0 + 8 * i + c_lo, g = ch >> 2;
          lo[i] = make_float2(0.f, 0.f); hi[i] = lo[i];
          if (g < P.Gout_store) {
            const float* o = reinterpret_cast<const float*>(P.out + ((size_t)b * P.Gout_store + g) * P.rows) + (ch & 3);
            if (ok_lo) lo[i] = *reinterpret_cast<const float2*>(o + (size_t)p_lo * 4);
            if (ok_hi) hi[i] = *reinterpret_cast<const float2*>(o + (size_t)p_hi * 4);
          }
        }
#pragma unroll
        for (int i = 0; i < NT / 8; ++i) stat_add<NT>(s_stat, cw, lane, 8 * i + c_lo, lo[i].x, lo[i].y, hi[i].x, hi[i].y);
      }
    }
    stat_flush<NT>(P, s_stat, et, b, n0);
  }
}

// weights: from the SIMT packing wt[tap][cin_pad][cout_pad] to
//   w[nt][chunk][tg][t][kg][n][4]  (tf32-rounded, round-to-nearest-away like cuDNN's conversion)
__global__ void k_pack_tc(const float* __restrict__ wt, float* __restrict__ w, int ntaps, int cin_pad, int cout_pad,
                          int NT, int nchunk, int ntg, int tpg, int KG) {
  size_t total = (size_t)(cout_pad / NT) * nchunk * ntg * tpg * KG * NT * 4;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int jj = i % 4;
  size_t r = i / 4;
  int n = r % NT; r /= NT;
  int kg = r % KG; r /= KG;
  int t = r % tpg; r /= tpg;
  int tg = r % ntg; r /= ntg;
  int cc = r % nchunk; r /= nchunk;
  int nt = (int)r;
  int tap = tg * tpg + t;
  int ci = (cc * KG + kg) * 4 + jj;
  float v = 0.0f;
  if (ci < cin_pad) v = wt[((size_t)tap * cin_pad + ci) * cout_pad + nt * NT + n];
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  w[i] = __uint_as_float(u);
}
// the FP16 packing of the same weights for the FP16 kernels: w16[nt][chunk][tg][t][kg][n][8], rounded to nearest even
// (what tensor.half() does); a 16-byte group holds 8 input channels
__global__ void k_pack_tc16(const float* __restrict__ wt, __half* __restrict__ w, int ntaps, int cin_pad, int cout_pad,
                            int NT, int nchunk, int ntg, int tpg, int KG) {
  size_t total = (size_t)(cout_pad / NT) * nchunk * ntg * tpg * KG * NT * 8;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  int jj = i % 8;
  size_t r = i / 8;
  int n = r % NT; r /= NT;
  int kg = r % KG; r /= KG;
  int t = r % tpg; r /= tpg;
  int tg = r % ntg; r /= ntg;
  int cc = r % nchunk; r /= nchunk;
  int nt = (int)r;
  int tap = tg * tpg + t;
  int ci = (cc * KG + kg) * 8 + jj;
  float v = 0.0f;
  if (ci < cin_pad) v = wt[((size_t)tap * cin_pad + ci) * cout_pad + nt * NT + n];
  w[i] = __float2half_rn(v);
}

}  // namespace tc

// channel groups (16 bytes: 4 fp32 or 8 fp16 channels) per chunk of a convolution with G input groups
static int conv_tc_kg(int ntaps, int NT, int G) {
  int KG = (ntaps == 27 && NT > 64) ? 4 : 8;
  if (G < KG) KG = (G <= 2) ? 2 : ((G <= 4) ? 4 : 8);
  return KG;
}

// The tiling of a convolution: decided here once, stored in w.tc with the packing laid out for it, and read by
// conv_tc_run, ygemm and sa_fused.  Adds the step that packs w.wt into w.tc.w.
int conv_tc_prepare(Model* m, ConvW& w) {
  w.tc = ConvTcW();
  if (!(w.ntaps == 27 || w.ntaps == 1)) return 0;
  if (w.cout_pad < 32 || w.cout_pad % 32) return 0;      // the kernel is instantiated for N = 32, 64, 96, 128
  ConvTcW t;
  t.NT = w.cout_pad < 128 ? w.cout_pad : 128;
  if (w.cout_pad % t.NT) return 0;
  t.ntg = w.ntaps == 27 ? 3 : 1;
  t.tpg = w.ntaps == 27 ? 9 : 1;
  const int G = w.cin_pad / 4;
  // 3x3x3: 32-channel chunks (36 wgmmas per activation stage) for N <= 64 -- the per-stage barrier
  // round trip is amortised over more MMAs -- and 16-channel chunks for N = 128, where the 9-tap
  // weight slab (2 x 72 KB) leaves room for a 16-channel ring only.
  // 1x1: 32-channel chunks.
  t.KG = conv_tc_kg(w.ntaps, t.NT, G);
  t.nchunk = (G + t.KG - 1) / t.KG;
  const size_t total = (size_t)(w.cout_pad / t.NT) * t.nchunk * t.ntg * t.tpg * t.KG * t.NT * 4;
  LION_TRY(m->dmalloc(&t.w, total));
  w.tc = t;
  m->repack.push_back([t, wt = w.wt, ntaps = w.ntaps, cin_pad = w.cin_pad, cout_pad = w.cout_pad, total] {
    tc::k_pack_tc<<<(unsigned)cdivz(total, 256), 256>>>(wt, t.w, ntaps, cin_pad, cout_pad, t.NT, t.nchunk, t.ntg, t.tpg, t.KG);
  });
  return 0;
}

// The FP16 tiling of a 3x3x3 convolution that has a TF32 one: the same record in 16-byte groups (C/8 of them), so KG,
// the chunk bytes, the rings, the block groups and the work distribution follow from bytes exactly as for TF32.  Only
// the cases the second convolutions of the PVConvs use are compiled (conv_tc_run), and only those are served: Cin = Cout =
// 32, 64 or 128 (N = 32, 64, 128 with KG = 4, 8, 4).  Allocates and adds the packing step; the caller runs it.  A
// convolution the FP16 kernels do not serve keeps tc16.w == nullptr.
int conv_tc_prepare_f16(Model* m, ConvW& w) {
  if (w.tc16.w || !w.tc.w || w.ntaps != 27 || w.cin_pad != w.cout_pad || w.cout != w.cout_pad) return 0;
  if (!(w.cout_pad == 32 || w.cout_pad == 64 || w.cout_pad == 128)) return 0;
  ConvTcW t = w.tc;
  const int G = w.cin_pad / 8;
  t.KG = conv_tc_kg(w.ntaps, t.NT, G);
  t.nchunk = (G + t.KG - 1) / t.KG;
  if (!((t.NT == 32 && t.KG == 4) || (t.NT == 64 && t.KG == 8) || (t.NT == 128 && t.KG == 4))) return 0;
  const size_t total = (size_t)(w.cout_pad / t.NT) * t.nchunk * t.ntg * t.tpg * t.KG * t.NT * 8;
  __half* w16 = nullptr;
  LION_TRY(m->dmalloc(&w16, total));
  t.w = reinterpret_cast<float*>(w16);
  w.tc16 = t;
  m->repack.push_back([t, w16, wt = w.wt, ntaps = w.ntaps, cin_pad = w.cin_pad, cout_pad = w.cout_pad, total] {
    tc::k_pack_tc16<<<(unsigned)cdivz(total, 256), 256>>>(wt, w16, ntaps, cin_pad, cout_pad, t.NT, t.nchunk, t.ntg, t.tpg, t.KG);
  });
  return 0;
}

// whether conv_tc_run computes this 3x3x3 convolution on row tiles, the only tiling that takes class-valued blocks
bool conv_tc_row_tiles_3x3(const ConvW& w) { return w.tc.w && w.ntaps == 27 && w.tc.NT <= 64; }

bool conv_tc_usable(const ConvW& w, const ConvGeom& geo) {
  if (!w.tc.w) return false;
  if (geo.ntaps != w.ntaps) return false;
  return true;
}

int conv_tc_run(Ctx* c, const ConvW& w, const float4* in, int Gin, float4* out, int Gout_store, double* ssum, double* ssq,
                const ConvGeom& geo, int B, float* pool_mm, bool f16) {
  tc::Params P{};
  if (f16 && !w.tc16.w) { set_error("conv_tc: no FP16 packing of this convolution"); return LION_ERR_STATE; }
  const ConvTcW& T = f16 ? w.tc16 : w.tc;   // f16: the input is [C/8][rows][8] halves
  if (pool_mm && (w.ntaps != 1 || geo.p_begin != 0 || geo.p_end != geo.rows || geo.rows % 128)) {
    set_error("conv_tc: the pooled epilogue needs a 1x1 convolution over a multiple of 128 rows"); return LION_ERR_ARG;
  }
  P.pool_mm = pool_mm;
  const int NT = T.NT, KG = T.KG, tpg = T.tpg;
  P.in = in; P.w = T.w; P.bias = w.bias; P.out = out; P.ssum = ssum; P.ssq = ssq;
  P.Gin = Gin; P.Gout_store = Gout_store; P.cout_pad = w.cout_pad;
  P.rows = geo.rows; P.p_begin = geo.p_begin; P.p_end = geo.p_end;
  P.ntg = T.ntg; P.tpg = tpg; P.KG = KG; P.nchunk = T.nchunk; P.NT = NT;
  const int slab_bytes = tpg * KG * NT * 16;     // the weights of one (channel chunk, x-plane)
  P.B = B;
  P.occ = geo.occ; P.occ_stride = geo.occ_stride;
  P.cls_flag = geo.cls_flag; P.cls_stride = geo.cls_stride; P.cls = geo.cls; P.cls_store = geo.cls_store ? 1 : 0;
  const size_t fixed = tc::smem_fixed(NT, tpg);
  // 3x3x3 with N = 128 runs on interior blocks (BLK); its chunking (16 channels) and so every output's accumulation
  // order are those of the row tiles.  N <= 64 keeps the 128-row tiles: its 32-channel chunks leave no room for a
  // block group's window beside the two weight slabs, and 16-channel chunks would reorder every output's sums.
  const bool blk = w.ntaps == 27 && NT == 128;
  // the 128-row tiles of [p_begin, p_end): the work space of row-tile kernels, and of the statistics pass (k_conv_stats)
  const int ntile_rows = cdiv(geo.p_end - geo.p_begin, 128);
  int ntile;
  P.halo = 0;
  if (w.ntaps == 27) {
    const int rp = geo.rp, r = rp - 2;
    for (int dx = 0; dx < 3; ++dx) P.tg_off[dx] = (dx - 1) * rp * rp;
    for (int dy = 0; dy < 3; ++dy) for (int dz = 0; dz < 3; ++dz) P.tap_off[dy * 3 + dz] = (dy - 1) * rp + (dz - 1);
    P.r = r; P.rp = rp;
  } else {
    P.tg_off[0] = 0; P.tap_off[0] = 0;
  }
  const int n_tiles_n = w.cout_pad / NT;
  if (blk) {
    const int rp = P.rp, r = P.r;
    P.nzb = cdiv(r, 8); P.npl = P.nzb * P.nzb; P.nblk = r * P.npl;
    // A group's window is its blocks' rows plus every tap's neighbours: from (y0-1, z0-1) of its first block to
    // (y0+8, z0+8) of its last; the largest sets the stage.  At N = 128 that is two whole x-planes at r = 8 (200 rows)
    // and 8 y-lines x 16 z at r = 16 (180 rows) for 2-block groups, one whole haloed x-plane (324 rows) for 4-block
    // groups at r = 16.
    auto window_rows = [&](int ib) {
      int wrows = 0;
      for (int f = 0; f < P.nblk; f += ib) {
        const int l = std::min(f + ib, P.nblk) - 1;
        wrows = std::max(wrows, tc::block_row(l, rp, P.nzb, P.npl) - tc::block_row(f, rp, P.nzb, P.npl) + 9 * rp + 10);
      }
      return wrows;
    };
    // Blocks per group: one per warpgroup, or two (two accumulator sets per thread), which doubles the MMAs of every
    // weight slab and A stage and halves the per-slab barrier round trips, copy latencies and item epilogues.  4-block
    // groups are taken while there are still as many groups as SMs, and while their window leaves one A stage more than
    // the 2 weight slabs (each slab consumes one A stage).  At B = 32 that is r = 16 (512 groups, 3 A stages), not
    // r = 8 (64 groups would idle half the SMs).
    const long long a_room2 = 227LL * 1024 - (long long)fixed - 2LL * slab_bytes;
    const bool four = (long long)n_tiles_n * B * cdiv(P.nblk, 4) >= c->num_sms && a_room2 / (KG * window_rows(4) * 16) >= 3;
    P.ib = four ? 4 : 2;
    P.stage_rows = window_rows(P.ib);
    ntile = cdiv(P.nblk, P.ib);
    P.G = 1;
  } else {
    if (w.ntaps == 27) P.halo = P.rp + 1;
    P.stage_rows = 128 + 2 * P.halo;
    ntile = ntile_rows;
    // row tiles per work item: as many as the accumulator registers hold (the weight slab of a stage is then shared by
    // that many MMA groups); parallelism does not depend on G -- the kernel cuts the flat tile space into equal ranges per CTA
    P.G = tc::tiles_per_item(NT);
  }
  P.ntile = ntile;
  P.a_stage_bytes = KG * P.stage_rows * 16;
  // Round-based items (sched 1) for 3x3x3 grids whose input is well beyond the L2: the three x-plane sweeps of a tile then
  // hit the L2 instead of re-reading DRAM.  Measured on an H100 SXM (400 W, B = 32, kernel alone, sched 0 / 1 alternated
  // twice): every grid above 1.6x the 50 MB L2 runs faster with rounds (64 ch @ 32^3, 322 MB: 7-9 %; 32 ch @ 32^3,
  // 161 MB: 3-4 %; the two 128-channel grids @ 16^3, 95 MB: 5-8 %); below it the two are within about 2 % either way
  // (one pair of runs of one 25 MB grid excepted), and one contiguous range per CTA is kept.
  const double in_bytes = (double)B * Gin * geo.rows * 16.0;
  P.sched = w.ntaps == 27 && in_bytes > 1.6 * c->l2_bytes ? 1 : 0;
  // The rings for weight stages of tps taps each; returns the A ring's depth, 0 if it cannot hold 2 stages.
  //   * Weight ring.  Whole slabs: 2.  A block group takes one A stage per weight slab, so the copies run ahead of the
  //     tensor cores by as many slabs as the weight ring holds: deepen it to 3-4 while at least 4 A stages (and one per
  //     slab) still fit -- under the side-stream cap when one is set.  Row tiles share a slab among up to 4 tiles and
  //     keep 2.  3-tap parts: 4, the 3 parts of the slab in use and 1 in flight.
  //   * A ring: what the weight ring and the fixed part leave of 227 KB (at most MAX_A_STAGES).  Sharing an SM with the
  //     side stream: FPS and the neighbour searches run on the side stream during the first ~1 ms of a step (32 CTAs x
  //     <= 26 KB of shared memory, latency-bound); a persistent convolution CTA that claims all 227 KB cannot become
  //     resident on their SMs, and with the static item split the whole convolution then takes two waves
  //     (tools/timeline_step.py shows it).  While the caller flags side-stream work (Ctx::conv_smem_cap) the ring gives
  //     up a slot or two -- never below 4 -- and the side kernels opt into the maximum shared-memory carve-out, because
  //     an SM only hosts kernels of one carve-out at a time.
  auto ring = [&](int tps, int& b_stages) -> int {
    const long long stage = (long long)slab_bytes / tpg * tps;
    b_stages = tps == tpg ? 2 : tc::MAX_B_STAGES;
    if (blk && tps == tpg) {
      const long long limit = (c->conv_smem_cap > 0 ? c->conv_smem_cap : 227LL * 1024) - (long long)fixed;
      while (b_stages < tc::MAX_B_STAGES && (limit - (b_stages + 1) * stage) / P.a_stage_bytes >= std::max(4, b_stages + 1))
        ++b_stages;
    }
    int a_stages = (int)((227LL * 1024 - (long long)fixed - b_stages * stage) / P.a_stage_bytes);
    if (c->conv_smem_cap > 0 && a_stages >= 5) {
      const int capped = (int)(((long long)c->conv_smem_cap - (long long)fixed - b_stages * stage) / P.a_stage_bytes);
      if (capped >= 4 && capped < a_stages) a_stages = capped;
    }
    a_stages = std::min(a_stages, tc::MAX_A_STAGES);
    return a_stages >= 2 ? a_stages : 0;
  };
  // Weight stages: whole slabs (tpg taps), or -- block groups -- each slab streamed as 3 parts of 3 taps (taps 3s ..
  // 3s+2 are one contiguous run of the packing), which shrinks the weight ring and leaves the A ring the room: at B = 32
  // 5 A stages instead of 3 beside the weight ring at r = 16 (4-block groups) and 9 instead of 5 at r = 8.  Parts are
  // taken when they deepen the A ring and it still holds G + 1 = 2 windows.  No deadlock: producer and consumers walk
  // the same order (a slab's first part, its item's A stages, its other parts), and every release the producer waits
  // for needs only stages copied before it -- a part goes back after the group that follows its last group, an A stage
  // after the group that follows its last part's group, and a ring of >= G + 1 stages lets the producer copy that
  // group's stage first.  Each output's products and their order are those of whole slabs (taps 0-8 of each chunk and
  // x-plane, k-steps in order), so the choice changes no bit of any output.
  //   Row tiles (N <= 64) keep whole slabs.  Their consumers wait on full A stages for 3.5 % of their time at r = 32
  // and 6.6 % at r = 16 (clock64 around the waits, 64 -> 64, B = 32), and 3-tap parts -- a commit group of 12 instead
  // of 36 wgmmas per tile, a barrier round trip per part -- measured 20-25 % slower there.  The 4-block groups at r = 16
  // waited 9 % of their time on A stages and 16 % on weight slabs; see DESIGN 4.1 for the numbers.
  int b_whole = 0, b_parts = 0;
  const int a_whole = ring(tpg, b_whole);
  const int a_parts = blk && !c->conv_whole_slabs ? ring(3, b_parts) : 0;
  const bool parts = a_parts > a_whole && a_parts >= P.G + 1;
  if (!parts && !a_whole) {
    set_error("conv_tc: shared memory cannot hold the operand pipeline (N=%d, KG=%d)", NT, KG); return LION_ERR_ARG;
  }
  P.tps = parts ? 3 : tpg;
  P.b_stage_bytes = slab_bytes / tpg * P.tps;
  P.b_stages = parts ? b_parts : b_whole;
  const int a_stages = parts ? a_parts : a_whole;
  P.a_stages = a_stages;
  const int b_stages = P.b_stages;
  // Occupancy skips need an A ring of two items' worth of row tiles.  A consumer hands the stage of its last MMA group
  // back at its next issue; on a shallower ring a run of skipped stages comes round to that stage first, and producer and
  // consumers wait for each other (4-tile items on the 6-stage ring of N = 32 with 32-channel chunks).  Without the flags
  // the all-zero slabs are multiplied instead, which adds exact zeros.  (Block groups retire every slab.)
  if (!blk && P.occ && a_stages < 2 * P.G) P.occ = nullptr;
  // Class-valued blocks (Params::cls_flag): the producer copies, and the consumers wait for, the A stages of the tiles
  // with a computed block only.  A warpgroup with a class-valued block in an item retires its MMAs at the end of every
  // slab, so it holds an A stage only while it waits for the stages of the same slab's later tiles, fewer than G: an A
  // ring of G stages cannot deadlock (test_conv2_const_skip_cpu.py simulates the protocol).  On a shallower ring every
  // block is computed, which gives the same bits.
  if (P.cls_flag && (blk || w.ntaps != 27 || P.occ || 2 * ntile > P.cls_stride)) {
    set_error("conv_tc: class-valued blocks are for 3x3x3 row tiles of a dense input"); return LION_ERR_ARG;
  }
  if (a_stages < P.G) P.cls_flag = nullptr;
  size_t smem = (size_t)a_stages * P.a_stage_bytes + (size_t)b_stages * P.b_stage_bytes + fixed;
  if (smem > 227 * 1024) { set_error("conv_tc: %zu bytes of shared memory needed", smem); return LION_ERR_ARG; }
  // persistent, at most one CTA per SM: the fewest CTAs that still reach the minimal maximum of tiles per CTA
  // (224 tiles on 132 SMs: 112 CTAs x 2 tiles, not 132 CTAs x 1-2 -- every CTA streams the whole weight tensor from L2
  // once per item, and the r = 8 layers are bound by exactly that)
  auto grid_for = [&](int nt_per_shape) {
    long long n_units = (long long)nt_per_shape * n_tiles_n * B;
    long long per_cta = (n_units + c->num_sms - 1) / c->num_sms;
    return (int)((n_units + per_cta - 1) / per_cta);
  };
  const int grid = grid_for(ntile);
  // block groups: the GroupNorm statistics come from k_conv_stats, over the row tiles' items
  tc::Params S = P;
  if (blk && ssum) {
    P.ssum = nullptr; P.ssq = nullptr;
    S.ntile = ntile_rows; S.G = tc::tiles_per_item(NT);
  }
  auto stats = [&]() -> int {
    if (!(blk && ssum)) return 0;
    LION_LAUNCH(c, tc::k_conv_stats<128>, grid_for(ntile_rows), 256, 0, S);
    return check_launch(c, "conv_tc stats");
  };
  const int bpw = blk ? P.ib / 2 : 1;
  c->conv_group_blocks = blk ? P.ib : 0;
  c->conv_stage_taps = P.tps;
#define CONV_TC_CASE_OP(kg, tpg_, nt_, blk_, bpw_, tps_, op)                                              \
  if (f16 == std::is_same<op, __half>::value && KG == kg && tpg == tpg_ && NT == nt_ && blk == blk_ && bpw == bpw_ && P.tps == tps_) { \
    static DevOnce attr_once;                                                                             \
    if (attr_once.need()) {                                                                               \
      LION_CHECK_CUDA(cudaFuncSetAttribute(tc::k_conv_tc<kg, tpg_, nt_, blk_, bpw_, tps_, op>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)); \
    }                                                                                                     \
    LION_LAUNCH(c, (tc::k_conv_tc<kg, tpg_, nt_, blk_, bpw_, tps_, op>), grid, tc::conv_threads(bpw_), smem, P); \
    LION_TRY(check_launch(c, "conv_tc"));                                                                 \
    return stats();                                                                                       \
  }
#define CONV_TC_CASE(kg, tpg_, nt_, blk_, bpw_, tps_) CONV_TC_CASE_OP(kg, tpg_, nt_, blk_, bpw_, tps_, float)
#define CONV_TC_NT(kg, tpg_) CONV_TC_CASE(kg, tpg_, 32, false, 1, tpg_) CONV_TC_CASE(kg, tpg_, 64, false, 1, tpg_) CONV_TC_CASE(kg, tpg_, 96, false, 1, tpg_)
#define CONV_TC_BLK(kg, bpw_) CONV_TC_CASE(kg, 9, 128, true, bpw_, 9) CONV_TC_CASE(kg, 9, 128, true, bpw_, 3)
  CONV_TC_NT(2, 1) CONV_TC_NT(4, 1) CONV_TC_NT(8, 1) CONV_TC_NT(2, 9) CONV_TC_NT(4, 9) CONV_TC_NT(8, 9)
  CONV_TC_CASE(2, 1, 128, false, 1, 1) CONV_TC_CASE(4, 1, 128, false, 1, 1) CONV_TC_CASE(8, 1, 128, false, 1, 1)
  CONV_TC_BLK(2, 1) CONV_TC_BLK(4, 1) CONV_TC_BLK(2, 2) CONV_TC_BLK(4, 2)
  // FP16 operands: the second convolutions of the PVConvs only (conv_tc_prepare_f16)
  CONV_TC_CASE_OP(4, 9, 32, false, 1, 9, __half) CONV_TC_CASE_OP(8, 9, 64, false, 1, 9, __half)
  CONV_TC_CASE_OP(4, 9, 128, true, 1, 9, __half) CONV_TC_CASE_OP(4, 9, 128, true, 1, 3, __half)
  CONV_TC_CASE_OP(4, 9, 128, true, 2, 9, __half) CONV_TC_CASE_OP(4, 9, 128, true, 2, 3, __half)
#undef CONV_TC_NT
#undef CONV_TC_BLK
#undef CONV_TC_CASE
#undef CONV_TC_CASE_OP
  set_error("conv_tc: no %s kernel for N=%d, KG=%d, %d taps, %d per weight stage", f16 ? "FP16" : "TF32", NT, KG, tpg, P.tps);
  return LION_ERR_ARG;
}

}  // namespace lion

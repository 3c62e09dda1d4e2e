// lion_b200 -- first half of the SPARSE first convolution of a PVConv (sm_90a).
//
// A PVConv's first 3x3x3 convolution reads a voxel grid with at most N occupied voxels (2048 of 32768 at r = 32).
// Instead of 27 dense taps over all r^3 positions, the occupied voxels' features x[v] (compact list, k_scatter_compact)
// are multiplied by all 27 taps at once,
//     y[v][t * C + c] = sum_ci  W[t][ci][c] * x[v][ci]                       (this file: one GEMM, K = Cin, 27*C columns)
// and every output voxel then sums the rows y[v(p + off(t))][t] of its occupied neighbours (k_sparse_conv_gather,
// packed_kernels.cuh).  16x fewer FLOPs at r = 32; the cost is streaming y once out and once in.
//
// One GEMM: the voxels are the A operand (M = 128 voxel rows per block, K-major = the packed [C/4][rows][4] layout as it
// lies in HBM), the weights the B operand (N = 128 tap-channels of one n-tile).  One CTA = two warpgroups (64 voxel rows
// each), one n-tile, a strided range of 128-row blocks; operands by cp.async.bulk; the next block's voxels are requested
// as soon as the MMAs of the current one retire, i.e. under the epilogue.  Every store of a warp writes 8 rows x 32
// contiguous bytes of y.
#include "common.cuh"
#include "model.cuh"
#include "wgmma.cuh"
#include <cstdlib>

namespace lion {
namespace spc {

using namespace sm90;

constexpr int ROWS = 128;     // voxel rows per block (two m64 warpgroups)

struct Params {
  const float4* x;       // compact voxel features, PF [B][G][N]
  const float* w;        // conv_tc packing of the wide 1x1 convolution: [n-tile][G][128][4], tf32-rounded
  float* y;              // [B][N][ld]
  const int* nocc;       // [B] occupied voxels per shape (rows beyond are never read back: skipped)
  int G, N, B, ld, blocks_per_shape, nblocks;
};

__global__ void __launch_bounds__(256, 2) k_ygemm(Params P) {
  extern __shared__ __align__(128) uint8_t smem[];
  float4* sW = (float4*)smem;                              // [G][128]
  float4* sX = sW + (size_t)P.G * 128;                     // [G][ROWS]
  uint64_t* bars = (uint64_t*)(sX + (size_t)P.G * ROWS);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nt = blockIdx.x;
  const uint32_t bar_w = smem_u32(bars), bar_x = smem_u32(bars + 1);
  if (tid == 0) {
    mbar_init(bar_w, 1);
    mbar_init(bar_x, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  auto block_rows = [&](int rb, int& b, int& r0) -> int {       // rows of block rb that matter (0 = skip)
    b = rb / P.blocks_per_shape;
    r0 = (rb % P.blocks_per_shape) * ROWS;
    int n = min(P.nocc ? __ldg(P.nocc + b) : P.N, P.N) - r0;
    return n < 0 ? 0 : (n > ROWS ? ROWS : n);
  };
  auto load_x = [&](int b, int r0, int nrows) {                 // thread 0 only
    const uint32_t bytes = (uint32_t)nrows * 16u;
    mbar_expect_tx(bar_x, bytes * (uint32_t)P.G);
    for (int g = 0; g < P.G; ++g)
      bulk_g2s(smem_u32(sX + (size_t)g * ROWS), P.x + ((size_t)b * P.G + g) * P.N + r0, bytes, bar_x);
  };
  // the first block this CTA owns that holds occupied voxels
  int rb = blockIdx.y;
  int b = 0, r0 = 0, nrows = 0;
  while (rb < P.nblocks && (nrows = block_rows(rb, b, r0)) == 0) rb += gridDim.y;
  if (tid == 0) {
    const uint32_t wbytes = (uint32_t)P.G * 128u * 16u;
    mbar_expect_tx(bar_w, wbytes);
    bulk_g2s(smem_u32(sW), P.w + (size_t)nt * P.G * 128 * 4, wbytes, bar_w);
    if (rb < P.nblocks) load_x(b, r0, nrows);
  }
  // (rows a partial block does not load hold stale bytes: output rows are independent and those rows are never stored)
  mbar_wait(bar_w, 0);
  uint32_t phase = 0;
  const int wg = warp >> 2, wq = warp & 3;
  const int r_lo = 64 * wg + 16 * wq + (lane >> 2);             // this thread's rows r_lo, r_lo + 8 of a block,
  const int c_lo = nt * 128 + 2 * (lane & 3);                   // its columns c_lo + 8 i + {0, 1}
  const uint64_t ad = make_desc(smem_u32(sX) + wg * 64 * 16, ROWS * 16, 128), bd = make_desc(smem_u32(sW), 128 * 16, 128);
  while (rb < P.nblocks) {
    mbar_wait(bar_x, phase);
    float acc[64];
    wg_fence();
    for (int ks = 0; ks < P.G / 2; ++ks)
      wgmma_tf32<128>(acc, ad + (uint64_t)((ks * 2 * ROWS * 16) >> 4), bd + (uint64_t)((ks * 2 * 128 * 16) >> 4), ks);
    wg_commit();
    wg_wait<0>();
    fence_regs<64>(acc);
    __syncthreads();                                            // both warpgroups have read the voxel buffer
    // the voxel buffer is free again: request the next block now, under this block's epilogue
    const int cb = b, cr0 = r0, cn = nrows;
    int nb = rb + gridDim.y, b2 = 0, r2 = 0, n2 = 0;
    while (nb < P.nblocks && (n2 = block_rows(nb, b2, r2)) == 0) nb += gridDim.y;
    if (tid == 0 && nb < P.nblocks) load_x(b2, r2, n2);
    rb = nb; b = b2; r0 = r2; nrows = n2;
    // ---- epilogue
    const size_t ldb = (size_t)P.ld;
    float* y_lo = P.y + ((size_t)cb * P.N + cr0 + r_lo) * ldb + c_lo;
    float* y_hi = y_lo + 8 * ldb;
    const bool ok_lo = r_lo < cn, ok_hi = r_lo + 8 < cn;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (nt * 128 + 8 * i < P.ld) {                            // ld is a multiple of 32: whole 8-column blocks
        if (ok_lo) *reinterpret_cast<float2*>(y_lo + 8 * i) = make_float2(acc[4 * i], acc[4 * i + 1]);
        if (ok_hi) *reinterpret_cast<float2*>(y_hi + 8 * i) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
      }
    }
    phase ^= 1;
  }
}

}  // namespace spc

bool ygemm_usable(const ConvW& y) {
  return y.tc.w && y.ntaps == 1 && y.tc.NT == 128 && y.cin_pad % 8 == 0 && y.cin_pad <= 128 &&
         y.tc.nchunk * y.tc.KG == y.cin_pad / 4;
}

// y[b][v][0..ld) = x[b][v][:] * Wy for the first nocc[b] rows of every shape
int ygemm_run(Ctx* c, const ConvW& y, const float4* xc, float* out, int ld, const int* nocc, int B, int N) {
  if (ld % 32) { set_error("ygemm: row pitch %d is not a multiple of 32", ld); return LION_ERR_ARG; }
  spc::Params P{};
  P.x = xc; P.w = y.tc.w; P.y = out; P.nocc = nocc;
  P.G = y.tc.nchunk * y.tc.KG;              // group slots of the packing (>= cin_pad / 4; extra slots hold zero weights)
  if (P.G != y.cin_pad / 4) { set_error("ygemm: packed groups %d != input groups %d", P.G, y.cin_pad / 4); return LION_ERR_STATE; }
  P.N = N; P.B = B; P.ld = ld;
  P.blocks_per_shape = (N + spc::ROWS - 1) / spc::ROWS;
  P.nblocks = B * P.blocks_per_shape;
  const int n_tiles = y.cout_pad / 128;
  int slices = (2 * c->num_sms + n_tiles - 1) / n_tiles;
  if (slices > P.nblocks) slices = P.nblocks;
  if (slices < 1) slices = 1;
  const size_t smem = (size_t)P.G * (128 + spc::ROWS) * 16 + 64;
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(spc::k_ygemm, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    LION_CHECK_CUDA(cudaFuncSetAttribute(spc::k_ygemm, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  }
  if (smem > 200 * 1024) { set_error("ygemm: %d input channels do not fit shared memory", y.cin_pad); return LION_ERR_ARG; }   // > 113 KB: one CTA per SM
  LION_LAUNCH(c, spc::k_ygemm, dim3(n_tiles, slices), 256, smem, P);
  return check_launch(c, "ygemm");
}

}  // namespace lion

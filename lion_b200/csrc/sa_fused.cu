// lion_b200 -- fused set-abstraction MLP for sm_90a (PointNetSAModule, models/pvcnn2_ada.py:98-114, :140-164, :354-382):
//   ball-query gather -> 1x1 conv -> AdaGN + Swish -> 1x1 conv -> max over the 32 neighbours
// without ever materialising the [B, C, M, 32] tensors in HBM.  GroupNorm needs whole-tensor statistics before the
// activation that follows it, so the module is two passes over the same gather (the gathered rows come from an L2-resident
// feature tensor: 262 KB per shape at level 0):
//   pass 1: gather -> conv1 (wgmma, TF32) -> per-channel sum / sum of squares of layer 1.           Writes nothing else.
//   pass 2: gather -> conv1 -> AdaGN-1 + Swish in registers -> shared memory -> conv2 (wgmma) -> statistics of layer 2
//           + per (centre, channel) min and max over the 32 neighbours (conv_tc.cu: Params::pool_mm explains why the
//           two extremes are enough for max_i swish(affine(x_i))); k_act_pool_minmax finishes the module.
// One CTA = one warpgroup = 128 threads = 128 rows = 4 centres x 32 neighbours per tile; the rows are laid out so that
// warp w's accumulator fragments hold the 32 neighbours of one centre, so the max-pool is a warp reduction.  No warp
// specialisation: a CTA is a strictly serial gather -> MMA -> epilogue chain and the overlap comes from 4 CTAs per SM
// (50 KB of shared memory each).
// DRAM traffic of SA level 0 at B = 32: ~1.36 GB per step with the unfused kernels, indices + 2 x 17 MB with this one.
#include "common.cuh"
#include "model.cuh"
#include "wgmma.cuh"

namespace lion {
namespace saf {

using namespace sm90;

struct Params {
  const float4* feat;      // PF [B][GF][N]
  const float4* points;    // [B][N] xyz
  const float4* centers;   // [B][M]
  const int* nidx;         // [B][M][32]
  const float* w1;         // conv_tc packing [G1P][N1][4], tf32-rounded; groups >= 1+GF are zero
  const float* b1;         // [N1]
  const float* w2;         // [N1/4][N2][4]
  const float* b2;         // [N2]
  const float* scale1;     // [B][N1] folded AdaGN-1 (pass 2)
  const float* shift1;
  double* ssum; double* ssq;   // [B][stat_stride]: layer 1 (pass 1) or layer 2 (pass 2)
  int stat_stride;
  float* pool_mm;          // [B][N2/4][M][2][4]  (pass 2)
  int N, M, tiles_per_cta;
};

// one layer for the tile's 128 rows: two m64 halves, K = 4 * G channels from [G][128][4], weights [G][N][4]
template <int G, int N>
__device__ __forceinline__ void mma_layer(float (&acc)[2][N / 2], uint32_t a_addr, uint32_t b_addr) {
  wg_fence();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint64_t ad = make_desc(a_addr + h * 64 * 16, 128 * 16, 128), bd = make_desc(b_addr, N * 16, 128);
#pragma unroll
    for (int ks = 0; ks < G / 2; ++ks)        // K = 8 = two channel groups per wgmma
      wgmma_tf32<N>(acc[h], ad + (uint64_t)((ks * 2 * 128 * 16) >> 4), bd + (uint64_t)((ks * 2 * N * 16) >> 4), ks);
  }
  wg_commit();
  wg_wait<0>();
  fence_regs<N / 2>(acc[0]);
  fence_regs<N / 2>(acc[1]);
}

// GF feature groups (+1 coordinate group, padded to an even count G1), N1 / N2 output channels of the two layers
template <int GF, int N1, int N2, int PASS>
__global__ void __launch_bounds__(128, 4) k_sa_fused(Params P) {
  constexpr int G1 = (GF + 1 + 1) & ~1;        // groups of the layer-1 operand (K = 4*G1, multiple of 8)
  constexpr int G2 = N1 / 4;
  constexpr int NS = PASS == 1 ? N1 : N2;      // channels whose statistics this pass accumulates
  static_assert(N1 % 16 == 0 && N2 % 16 == 0 && N1 + N2 <= 128 && G2 % 2 == 0, "unsupported fused SA shape");
  extern __shared__ __align__(128) uint8_t smem[];
  float4* sA1 = (float4*)smem;                               // [G1][128]
  float4* sA2 = sA1 + G1 * 128;                              // [G2][128]
  float4* sW1 = sA2 + G2 * 128;                              // [G1][N1]
  float4* sW2 = sW1 + G1 * N1;                               // [G2][N2]
  float* s_b1 = (float*)(sW2 + G2 * N2);                     // [N1]
  float* s_b2 = s_b1 + N1;                                   // [N2]
  float* s_sc = s_b2 + N2;                                   // [N1]
  float* s_sh = s_sc + N1;                                   // [N1]
  float* s_stat = s_sh + N1;                                 // [4 warps][2][NS] running partial sums of each warp
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tiles_per_shape = P.M / 4;
  const int ctas_per_shape = (tiles_per_shape + P.tiles_per_cta - 1) / P.tiles_per_cta;
  const int b = blockIdx.x / ctas_per_shape;
  const int tile_begin = (blockIdx.x % ctas_per_shape) * P.tiles_per_cta;
  const int tile_end = min(tile_begin + P.tiles_per_cta, tiles_per_shape);

  // weights / biases / folded affine of this shape; the zero padding group of A1
  for (int i = tid; i < G1 * N1; i += 128) sW1[i] = ((const float4*)P.w1)[i];
  if (PASS == 2) for (int i = tid; i < G2 * N2; i += 128) sW2[i] = ((const float4*)P.w2)[i];
  if (tid < N1) {
    s_b1[tid] = P.b1 ? P.b1[tid] : 0.0f;
    if (PASS == 2) { s_sc[tid] = P.scale1[(size_t)b * N1 + tid]; s_sh[tid] = P.shift1[(size_t)b * N1 + tid]; }
  }
  if (PASS == 2 && tid < N2) s_b2[tid] = P.b2 ? P.b2[tid] : 0.0f;
  for (int g = GF + 1; g < G1; ++g) sA1[g * 128 + tid] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int i = tid; i < 8 * NS; i += 128) s_stat[i] = 0.0f;

  // Tile rows are ordered so that warp w's accumulator fragments hold the 32 neighbours of centre w: shared-memory row
  // 64 h + 16 w + j is neighbour 16 h + j of centre w (h = m64 half).  This thread's fragment rows are j = lane / 4 and
  // lane / 4 + 8 of both halves, its columns 8 i + 2 (lane % 4) + {0, 1}.
  const int c_lo = 2 * (lane & 3);
  const float4* feat_b = P.feat + (size_t)b * GF * P.N;
  const float4* pts_b = P.points + (size_t)b * P.N;
  // GroupNorm partials of columns col, col + 1 over this warp's rows of the tile, added to the warp's slot in s_stat (reduced
  // per tile rather than kept per thread: the running sums would cost NS / 2 registers for the whole kernel)
  auto stat_add = [&](int col, float s0, float s1, float q0, float q1) {
    s0 = red8<0>(s0); s1 = red8<0>(s1); q0 = red8<0>(q0); q1 = red8<0>(q1);
    if (lane < 4) {
      float* st = s_stat + (warp * 2) * NS + col;
      st[0] += s0; st[1] += s1; st[NS] += q0; st[NS + 1] += q1;
    }
  };

  for (int tile = tile_begin; tile < tile_end; ++tile) {
    // ---- gather: thread = (centre tile*4 + warp, neighbour lane)
    const int centre = tile * 4 + warp;
    __syncthreads();                        // the previous tile's wgmmas and shared-memory readers are done
    {
      const int row = 64 * (lane >> 4) + 16 * warp + (lane & 15);
      const int k = __ldg(P.nidx + ((size_t)b * P.M + centre) * 32 + lane);
      const float4 c = __ldg(P.centers + (size_t)b * P.M + centre);
      const float4 p = __ldg(pts_b + k);
      float4 f[GF];
#pragma unroll
      for (int g = 0; g < GF; ++g) f[g] = __ldg(feat_b + (size_t)g * P.N + k);
      sA1[row] = make_float4(p.x - c.x, p.y - c.y, p.z - c.z, 0.0f);
#pragma unroll
      for (int g = 0; g < GF; ++g) sA1[(g + 1) * 128 + row] = f[g];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> wgmma operand reads
    __syncthreads();
    {
      float acc[2][N1 / 2];
      mma_layer<G1, N1>(acc, smem_u32(sA1), smem_u32(sW1));
      // ---- layer 1 out of the accumulators
#pragma unroll
      for (int i = 0; i < N1 / 8; ++i) {
        const int col = 8 * i + c_lo;
        float s0 = 0.0f, s1 = 0.0f, q0 = 0.0f, q1 = 0.0f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) v[e] = acc[h][4 * i + e] + s_b1[col + (e & 1)];
          if (PASS == 1) {
            s0 += v[0] + v[2]; s1 += v[1] + v[3];
            q0 += fmaf(v[0], v[0], v[2] * v[2]); q1 += fmaf(v[1], v[1], v[3] * v[3]);
          } else {
            // AdaGN-1 + Swish, rounded to TF32 exactly like k_act_rows does for a convolution's input
#pragma unroll
            for (int e = 0; e < 4; ++e) v[e] = tf32_rna(swishf(fmaf(v[e], s_sc[col + (e & 1)], s_sh[col + (e & 1)])));
            float* a2 = (float*)sA2 + (size_t)((col >> 2) * 128 + 64 * h + 16 * warp + (lane >> 2)) * 4 + (col & 3);
            *reinterpret_cast<float2*>(a2) = make_float2(v[0], v[1]);
            *reinterpret_cast<float2*>(a2 + 8 * 4) = make_float2(v[2], v[3]);
          }
        }
        if (PASS == 1) stat_add(col, s0, s1, q0, q1);
      }
    }
    if (PASS == 2) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      float acc[2][N2 / 2];
      mma_layer<G2, N2>(acc, smem_u32(sA2), smem_u32(sW2));
#pragma unroll
      for (int i = 0; i < N2 / 8; ++i) {
        const int col = 8 * i + c_lo;
        float mn[2], mx[2], su[2], sq[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float bias = s_b2[col + e];
          const float a = acc[0][4 * i + e] + bias, b0 = acc[0][4 * i + 2 + e] + bias;
          const float c = acc[1][4 * i + e] + bias, d = acc[1][4 * i + 2 + e] + bias;
          su[e] = (a + b0) + (c + d);
          sq[e] = fmaf(a, a, b0 * b0) + fmaf(c, c, d * d);
          mn[e] = red8<1>(fminf(fminf(a, b0), fminf(c, d)));
          mx[e] = red8<2>(fmaxf(fmaxf(a, b0), fmaxf(c, d)));
        }
        stat_add(col, su[0], su[1], sq[0], sq[1]);
        if (lane < 4) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int ch = col + e;
            float* dst = P.pool_mm + ((((size_t)b * (N2 / 4) + (ch >> 2)) * P.M + centre) * 2) * 4 + (ch & 3);
            dst[0] = mn[e]; dst[4] = mx[e];
          }
        }
      }
    }
  }
  // ---- statistics: warp partials -> CTA (fixed order: bit-reproducible) -> one fp64 atomic per channel
  __syncthreads();
  if (tid < NS) {
    float a = 0.0f, q = 0.0f;
#pragma unroll
    for (int w = 0; w < 4; ++w) { a += s_stat[(w * 2 + 0) * NS + tid]; q += s_stat[(w * 2 + 1) * NS + tid]; }
    atomicAdd(P.ssum + (size_t)b * P.stat_stride + tid, (double)a);
    atomicAdd(P.ssq + (size_t)b * P.stat_stride + tid, (double)q);
  }
}

template <int GF, int N1, int N2>
constexpr size_t smem_bytes() {
  constexpr int G1 = (GF + 2) & ~1, G2 = N1 / 4;
  return (size_t)(G1 * 128 + G2 * 128 + G1 * N1 + G2 * N2) * 16 + (size_t)(N1 + N2 + 2 * N1 + 8 * (N1 > N2 ? N1 : N2)) * 4;
}

}  // namespace saf

// shapes this file is instantiated for: (feature channels, layer-1 width, layer-2 width)
bool sa_fused_usable(const SABlk& s) {
  if (s.mlp.conv.size() != 2 || s.k != 32 || s.m % 4) return false;
  const ConvW &c1 = s.mlp.conv[0], &c2 = s.mlp.conv[1];
  if (!c1.tc.w || !c2.tc.w || c1.cout != c1.cout_pad || c2.cout != c2.cout_pad) return false;
  return s.cfeat == 32 && c1.cout == 32 && c2.cout == 64 && c1.tc.NT == 32 && c2.tc.NT == 64 && c1.tc.KG == 8 && c2.tc.KG == 8;
}

// pass 1 (scale1 == nullptr): layer-1 statistics; pass 2: layer-2 statistics + pooled min / max
int sa_fused_run(Ctx* c, const SABlk& s, const float4* feat, const float4* points, const float4* centers, const int* nidx,
                 const float* scale1, const float* shift1, double* ssum, double* ssq, int stat_stride, float* pool_mm,
                 int B, int N) {
  saf::Params P{};
  const ConvW &c1 = s.mlp.conv[0], &c2 = s.mlp.conv[1];
  P.feat = feat; P.points = points; P.centers = centers; P.nidx = nidx;
  P.w1 = c1.tc.w; P.b1 = c1.bias; P.w2 = c2.tc.w; P.b2 = c2.bias;
  P.scale1 = scale1; P.shift1 = shift1; P.ssum = ssum; P.ssq = ssq; P.stat_stride = stat_stride; P.pool_mm = pool_mm;
  P.N = N; P.M = s.m;
  // CTAs: ~4 per SM resident; aim at about two waves so that the tail is short and the weight loads amortise
  const int tiles = s.m / 4;
  int tpc = 1;
  while (tpc < 16 && (long long)B * ((tiles + tpc - 1) / tpc) > 8LL * c->num_sms) tpc <<= 1;
  P.tiles_per_cta = tpc;
  const int grid = B * ((tiles + tpc - 1) / tpc);
  constexpr size_t smem = saf::smem_bytes<8, 32, 64>();
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(saf::k_sa_fused<8, 32, 64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    LION_CHECK_CUDA(cudaFuncSetAttribute(saf::k_sa_fused<8, 32, 64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  }
  if (!scale1) LION_LAUNCH(c, (saf::k_sa_fused<8, 32, 64, 1>), grid, 128, smem, P);
  else LION_LAUNCH(c, (saf::k_sa_fused<8, 32, 64, 2>), grid, 128, smem, P);
  return check_launch(c, "sa_fused");
}

}  // namespace lion

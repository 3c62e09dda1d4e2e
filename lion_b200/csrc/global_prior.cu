// lion_b200 -- the global-latent prior (PriorSEDrop / PriorSEClip): a 2048-wide residual MLP
// with squeeze-excite cells evaluated on a handful of rows (B <= 64 shapes).
//
// Reference: models/score_sde/resnet.py:195-218 (Prior.forward), :60-90 (ResBlockSEDrop),
// :29-56 (ResBlockSEClip), :16-27 (SE), models/utils.py:16-31 (PositionalEmbedding).
// The work is weight streaming (309 MB of fp32 weights per step for 0.15 GFLOP/shape), so the
// kernel is a skinny GEMM: every weight is read once, coalesced, and applied to all B rows
// held in shared memory; bias / ReLU / residual / SE gate are fused into the epilogue.
#include "common.cuh"
#include "model.cuh"
#include "../../include/lion_b200.h"
#include <cstdlib>

namespace lion {

constexpr int GP_MAXB = 32;     // rows (shapes) per call
constexpr int GP_BT = 32;
constexpr int GP_KS = 256;      // K slice per block (split-K)
constexpr int GP_PITCH = GP_KS + 4;
constexpr int GP_WARPS = 8;
constexpr int GP_OW = 16;       // outputs per warp (processed two at a time)
constexpr int GP_OB = GP_WARPS * GP_OW;   // 128 outputs per block
constexpr int GP_MAXSPLIT = 16;

__device__ __forceinline__ float warp_transpose_sum32(float* v, int lane) {
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1) {
    bool upper = (lane & half) != 0;
#pragma unroll
    for (int i = 0; i < half; ++i) {
      float keep = upper ? v[i + half] : v[i];
      float send = upper ? v[i] : v[i + half];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, half);
    }
  }
  return v[0];
}

// Split-K skinny GEMM, phase 1:  part[ks][b][o] = sum_{k in slice ks} W[o][k] * (x[b][k] + add[b][k])
// grid = (O/128, K/256).  Warp-level mma.sync.m16n8k8 TF32 (the reference's cuDNN 1x1 convolutions
// run TF32 as well): A = 16 weight rows x 8 k, B = 8 k x 8 shapes.  With the operands swapped
// (M = 128 weight rows, N = 32 shapes) this is a legal tensor-core tile shape too, but the layer is bound by
// launch latency and weight streaming (0.15 GFLOP per shape), not by the tensor pipe.
//   * the block's weight tile [128 x 256] (128 KB) streams HBM -> shared memory with cp.async in
//     four 64-column commit groups, so the tensor work on group g overlaps the arrival of g+1;
//   * the activation slice [32 x 256] is staged once per block (rounded to TF32, round-to-nearest);
//   * row pitch 260 floats makes every fragment load bank-conflict free (bank = 4*row + col).
// Deterministic: partials are summed in a fixed order by k_gp_reduce.
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ uint32_t tf32_bits(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return u;
}
struct GpEpi {
  const float* bias; float* out; int out_stride; const float* mul; int mul_stride; const float* res; int res_stride; int act;
};
__global__ void __launch_bounds__(GP_WARPS * 32, 1)
k_gp_partial(const float* __restrict__ W, const float* __restrict__ x, int x_stride, const float* __restrict__ add,
             int add_stride, float* __restrict__ part, int B, int K, int O, GpEpi epi) {
  extern __shared__ __align__(16) float s_mem[];
  float* s_w = s_mem;                          // [GP_OB][GP_PITCH]
  float* s_x = s_mem + GP_OB * GP_PITCH;       // [GP_BT][GP_PITCH]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int k0 = blockIdx.y * GP_KS, kt = min(GP_KS, K - k0);
  const int o0 = blockIdx.x * GP_OB;
  // weights: 4 commit groups of 64 columns; chunk c of a group = (row, 16-byte column piece)
  const uint32_t s_w_addr = (uint32_t)__cvta_generic_to_shared(s_w);
#pragma unroll
  for (int g = 0; g < 4; ++g) {
#pragma unroll
    for (int u = 0; u < (GP_OB * 16) / (GP_WARPS * 32); ++u) {       // 128 rows x 16 pieces / 256 threads = 8
      int c = tid + u * (GP_WARPS * 32);
      int row = c >> 4, piece = c & 15;
      int col = g * 64 + piece * 4;
      if (o0 + row < O && col < kt)
        cp_async16(s_w_addr + (uint32_t)(row * GP_PITCH + col) * 4u, W + (size_t)(o0 + row) * K + k0 + col);
      else   // keep out-of-range rows / columns finite: they meet zero activations or unused outputs
        *reinterpret_cast<float4*>(s_w + row * GP_PITCH + col) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  // activations (+ add), rounded to TF32
  {
    constexpr int PER_THREAD = GP_BT * (GP_KS / 4) / (GP_WARPS * 32);      // 8
    float4 v[PER_THREAD];
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) {
      int i = tid + u * (GP_WARPS * 32);
      int b = i / (GP_KS / 4), k4 = i % (GP_KS / 4);
      v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < B && k4 * 4 < kt) {
        v[u] = *reinterpret_cast<const float4*>(x + (size_t)b * x_stride + k0 + k4 * 4);
        if (add) {
          float4 a = *reinterpret_cast<const float4*>(add + (size_t)b * add_stride + k0 + k4 * 4);
          v[u].x += a.x; v[u].y += a.y; v[u].z += a.z; v[u].w += a.w;
        }
      }
    }
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) {
      int i = tid + u * (GP_WARPS * 32);
      int b = i / (GP_KS / 4), k4 = i % (GP_KS / 4);
      float4 r = make_float4(__uint_as_float(tf32_bits(v[u].x)), __uint_as_float(tf32_bits(v[u].y)),
                             __uint_as_float(tf32_bits(v[u].z)), __uint_as_float(tf32_bits(v[u].w)));
      *reinterpret_cast<float4*>(s_x + b * GP_PITCH + k4 * 4) = r;
    }
  }
  const int g8 = lane >> 2, t4 = lane & 3;
  float acc[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[n][i] = 0.0f;
  const float* wa = s_w + (wid * 16 + g8) * GP_PITCH + t4;       // rows g8 / g8+8 of this warp's 16 outputs
  const float* xb = s_x + g8 * GP_PITCH + t4;                    // shape g8 of each 8-shape tile
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    if (g == 0) asm volatile("cp.async.wait_group 3;" ::: "memory");
    else if (g == 1) asm volatile("cp.async.wait_group 2;" ::: "memory");
    else if (g == 2) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    if (g * 64 < kt) {
#pragma unroll
      for (int kk = 0; kk < 64; kk += 8) {
        const int k = g * 64 + kk;
        uint32_t a0 = __float_as_uint(wa[k]), a1 = __float_as_uint(wa[8 * GP_PITCH + k]);
        uint32_t a2 = __float_as_uint(wa[k + 4]), a3 = __float_as_uint(wa[8 * GP_PITCH + k + 4]);
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          uint32_t b0 = __float_as_uint(xb[n * 8 * GP_PITCH + k]), b1 = __float_as_uint(xb[n * 8 * GP_PITCH + k + 4]);
          asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                       : "+f"(acc[n][0]), "+f"(acc[n][1]), "+f"(acc[n][2]), "+f"(acc[n][3])
                       : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
        }
      }
    }
  }
  // C fragment: c0,c1 -> (row g8, shapes 2*t4, 2*t4+1); c2,c3 -> (row g8+8, same shapes)
  float* pout = part + (size_t)blockIdx.y * B * O;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int o = o0 + wid * 16 + g8 + (i >= 2 ? 8 : 0);
      int b = n * 8 + 2 * t4 + (i & 1);
      if (b < B && o < O) pout[(size_t)b * O + o] = acc[n][i];
    }
  }
}

// phase 2: out[b][o] = epi( sum_ks part[ks][b][o] + bias[o] );  act: 0 none, 1 relu, 2 sigmoid;
// mul: result *= mul[b][o] (SE gate);  res: result += res[b][o] (residual shortcut)
__global__ void k_gp_reduce(const float* __restrict__ part, int nsplit, const float* __restrict__ bias, float* __restrict__ out,
                            int out_stride, const float* __restrict__ mul, int mul_stride, const float* __restrict__ res,
                            int res_stride, int B, int O, int act) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * O) return;
  int b = i / O, o = i % O;
  float v = 0.0f;
  for (int s = 0; s < nsplit; ++s) v += part[((size_t)s * B + b) * O + o];
  v += bias ? bias[o] : 0.0f;
  if (act == 1) v = fmaxf(v, 0.0f);
  else if (act == 2) v = 1.0f / (1.0f + expf(-v));
  if (mul) v *= mul[(size_t)b * mul_stride + o];
  if (res) v += res[(size_t)b * res_stride + o];
  out[(size_t)b * out_stride + o] = v;
}

// Two kernels per Linear rather than one persistent kernel: a cooperative form without split-K makes every CTA re-read the
// whole [32 x K] activation matrix (2x its weight bytes), and a cluster / distributed-shared-memory split-K form pays a
// chain of barrier -> load -> MMA -> cluster barrier -> reduce per Linear that is no shorter than two graph-node
// boundaries.  The evaluation is launch/latency-bound, well above its 309 MB weight-streaming bound.
// PositionalEmbedding (models/utils.py:16-31): fp32 frequencies exp(i * -log(1e4)/(half-1))
__global__ void k_gp_posemb(const float* __restrict__ t, const float* __restrict__ freqs, float* __restrict__ out,
                            int half, float scale) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < half; i += blockDim.x) {     // any embedding_dim, whatever the block size
    float e = __fmul_rn(__fmul_rn(t[b], scale), freqs[i]);
    out[(size_t)b * 2 * half + i] = sinf(e);
    out[(size_t)b * 2 * half + half + i] = cosf(e);
  }
}

struct GPLin { const float* w; const float* b; int K, O; };
struct GlobalPriorBlk {
  int D = 128, nf = 2048, emb = 128, ncell = 8, clip = 0, clip_dim = 512;
  float scale = 1.0f;
  float* d_freqs = nullptr;
  GPLin t0, t1, cmap, in, outl;
  struct Cell { GPLin c1, c2, se0, se2; };
  std::vector<Cell> cells;
};
void global_prior_free(GlobalPriorBlk* g) { delete g; }

// desc: [D, nf, emb_dim, ncell, clip, clip_dim, scale_bits]; params in state_dict order:
//   [clip_feat_mapping.w,b] temb_layer.0.w,b temb_layer.1.w,b input_layer.w,b
//   all_modules.k.{conv1.w,b conv2.w,b SE.fc.0.w SE.fc.2.w} output_layer.w,b
int global_prior_build(Model* m, Cursor& cur) {
  const std::vector<int>& d = m->desc;
  if (d.size() < 7) { set_error("global prior descriptor: [D, nf, emb, ncell, clip, clip_dim, scale_bits]"); return LION_ERR_ARG; }
  GlobalPriorBlk* g = new GlobalPriorBlk();
  m->gp = g;
  g->D = d[0]; g->nf = d[1]; g->emb = d[2]; g->ncell = d[3]; g->clip = d[4]; g->clip_dim = d[5];
  memcpy(&g->scale, &d[6], 4);
  auto lin = [&](GPLin& l, int K, int O, bool bias) { l.w = cur.next(); l.b = bias ? cur.next() : nullptr; l.K = K; l.O = O; };
  if (g->clip) lin(g->cmap, g->clip_dim, g->nf, true);
  lin(g->t0, g->emb, g->emb * 4, true);
  lin(g->t1, g->emb * 4, g->nf, true);
  lin(g->in, g->D, g->nf, true);
  g->cells.resize(g->ncell);
  for (auto& c : g->cells) {
    lin(c.c1, g->clip ? 2 * g->nf : g->nf, g->nf, true);
    lin(c.c2, g->nf, g->nf, true);
    lin(c.se0, g->nf, g->nf / 8, false);
    lin(c.se2, g->nf / 8, g->nf, false);
  }
  lin(g->outl, g->nf, g->D, true);
  if (cur.bad) { set_error("global prior: parameter list too short (%d given)", cur.n); return LION_ERR_ARG; }
  int half = g->emb / 2;
  std::vector<float> fr(half);
  float step = (float)(std::log(10000.0) / (half - 1));      // python float -> fp32 tensor multiply
  for (int i = 0; i < half; ++i) fr[i] = expf((float)i * -step);
  LION_TRY(m->dmalloc(&g->d_freqs, (size_t)half));
  LION_CHECK_CUDA(cudaMemcpy(g->d_freqs, fr.data(), half * sizeof(float), cudaMemcpyHostToDevice));
  return 0;
}

static int gp_linear(Ctx* c, const GPLin& l, const float* x, int xs, const float* add, int as, float* out, int os,
                     const float* mul, int ms, const float* res, int rs, int B, int act) {
  if (l.K % 4) { set_error("global prior: K=%d must be a multiple of 4 (16-byte loads)", l.K); return LION_ERR_ARG; }
  int nsplit = cdiv(l.K, GP_KS);
  if (nsplit > GP_MAXSPLIT) {
    set_error("global prior: K=%d needs %d K slices of %d, at most %d (K <= %d)", l.K, nsplit, GP_KS, GP_MAXSPLIT, GP_KS * GP_MAXSPLIT);
    return LION_ERR_ARG;
  }
  const size_t smem = (size_t)(GP_OB + GP_BT) * GP_PITCH * sizeof(float);
  static DevOnce attr_once;
  if (attr_once.need()) LION_CHECK_CUDA(cudaFuncSetAttribute(k_gp_partial, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  GpEpi epi{l.b, out, os, mul, ms, res, rs, act};
  size_t mk = c->mark();
  float* part = c->alloc_n<float>((size_t)nsplit * B * l.O);
  LION_LAUNCH(c, k_gp_partial, dim3(cdiv(l.O, GP_OB), nsplit), GP_WARPS * 32, smem, l.w, x, xs, add, as, part, B, l.K, l.O, epi);
  LION_LAUNCH(c, k_gp_reduce, cdiv(B * l.O, 256), 256, 0, part, nsplit, l.b, out, os, mul, ms, res, rs, B, l.O, act);
  c->release(mk);     // stream order makes reuse by the next layer safe
  return 0;
}

// lion_global_prior_probe: rows [b0, b0 + B) of a [.][w] caller buffer from `src` (row stride ss), real pass only
static int gp_tap(Ctx* c, float* dst, int b0, const float* src, int ss, int w, int B) {
  if (!dst || c->dry) return 0;
  LION_CHECK_CUDA(cudaMemcpy2DAsync(dst + (size_t)b0 * w, w * sizeof(float), src, ss * sizeof(float), w * sizeof(float), B,
                                    cudaMemcpyDeviceToDevice, c->stream));
  return 0;
}

// one chunk of <= 32 shapes (rows b0 .. b0 + B - 1 of the call): two kernels per Linear (split-K partial sums +
// deterministic reduce with fused epilogue)
static int global_prior_forward_layers(Model* m, const float* x, const float* t, const float* clip, float* out, int B,
                                       const GpRecord* rec, int b0) {
  GlobalPriorBlk* g = m->gp;
  Ctx* c = m->ctx;
  int nf = g->nf, tw = g->clip ? 2 * nf : nf;
  float* pe = c->alloc_n<float>((size_t)B * g->emb);
  float* t0 = c->alloc_n<float>((size_t)B * g->emb * 4);
  float* tadd = c->alloc_n<float>((size_t)B * tw);     // [temb | 0]: what is added to the cell input
  float* cat = c->alloc_n<float>((size_t)B * tw);      // [h | clip-mapped] (clip variant only)
  float* h = c->alloc_n<float>((size_t)B * nf);
  float* h2 = c->alloc_n<float>((size_t)B * nf);
  float* a = c->alloc_n<float>((size_t)B * nf);
  float* bb = c->alloc_n<float>((size_t)B * nf);
  float* s0 = c->alloc_n<float>((size_t)B * nf / 8);
  const GpRecord no_rec;
  const GpRecord& r = rec ? *rec : no_rec;
  LION_LAUNCH(c, k_gp_posemb, B, 64, 0, t, g->d_freqs, pe, g->emb / 2, g->scale);
  LION_TRY(gp_tap(c, r.pe, b0, pe, g->emb, g->emb, B));
  // temb_layer: two 1x1 convs, no nonlinearity in between (resnet.py:181-184)
  LION_TRY(gp_linear(c, g->t0, pe, g->emb, nullptr, 0, t0, g->emb * 4, nullptr, 0, nullptr, 0, B, 0));
  LION_TRY(gp_tap(c, r.t0, b0, t0, g->emb * 4, g->emb * 4, B));
  if (g->clip) LION_TRY(memset_async(c, tadd, 0, sizeof(float) * B * tw));
  LION_TRY(gp_linear(c, g->t1, t0, g->emb * 4, nullptr, 0, tadd, tw, nullptr, 0, nullptr, 0, B, 0));
  LION_TRY(gp_tap(c, r.temb, b0, tadd, tw, nf, B));
  // clip_feat_mapping output is concatenated behind temb (resnet.py:203-208) and reaches every
  // cell's conv1 un-added (ResBlockSEClip.forward, resnet.py:41-46)
  if (g->clip) {
    LION_TRY(gp_linear(c, g->cmap, clip, g->clip_dim, nullptr, 0, cat + nf, tw, nullptr, 0, nullptr, 0, B, 0));
    LION_TRY(gp_tap(c, r.cmap, b0, cat + nf, tw, nf, B));
  }
  LION_TRY(gp_linear(c, g->in, x, g->D, nullptr, 0, h, nf, nullptr, 0, nullptr, 0, B, 0));
  LION_TRY(gp_tap(c, r.h0, b0, h, nf, nf, B));
  for (size_t k = 0; k < g->cells.size(); ++k) {
    const auto& cell = g->cells[k];
    const GpRecord::Cell rc = r.cells ? r.cells[k] : GpRecord::Cell{};
    // conv1(x + t [| clip]) -> ReLU -> (dropout: identity in eval) -> conv2 -> ReLU -> SE -> + x
    if (g->clip) {
      if (!c->dry)
        LION_CHECK_CUDA(cudaMemcpy2DAsync(cat, tw * sizeof(float), h, nf * sizeof(float), nf * sizeof(float), B, cudaMemcpyDeviceToDevice, c->stream));
      LION_TRY(gp_linear(c, cell.c1, cat, tw, tadd, tw, a, nf, nullptr, 0, nullptr, 0, B, 1));
    } else {
      LION_TRY(gp_linear(c, cell.c1, h, nf, tadd, tw, a, nf, nullptr, 0, nullptr, 0, B, 1));
    }
    LION_TRY(gp_tap(c, rc.a, b0, a, nf, nf, B));
    LION_TRY(gp_linear(c, cell.c2, a, nf, nullptr, 0, bb, nf, nullptr, 0, nullptr, 0, B, 1));
    LION_TRY(gp_tap(c, rc.bb, b0, bb, nf, nf, B));
    LION_TRY(gp_linear(c, cell.se0, bb, nf, nullptr, 0, s0, nf / 8, nullptr, 0, nullptr, 0, B, 1));
    LION_TRY(gp_tap(c, rc.s, b0, s0, nf / 8, nf / 8, B));
    LION_TRY(gp_linear(c, cell.se2, s0, nf / 8, nullptr, 0, h2, nf, bb, nf, h, nf, B, 2));   // sigmoid(.) * bb + h
    LION_TRY(gp_tap(c, rc.h, b0, h2, nf, nf, B));
    float* tmp = h; h = h2; h2 = tmp;
  }
  LION_TRY(gp_linear(c, g->outl, h, nf, nullptr, 0, out, g->D, nullptr, 0, nullptr, 0, B, 0));
  return check_launch(c, "global_prior_forward");
}

int global_prior_forward(Model* m, const float* x, const float* t, const float* clip, float* out, int B, const GpRecord* rec) {
  GlobalPriorBlk* g = m->gp;
  Ctx* c = m->ctx;
  if (g->clip && !clip) { set_error("global prior: this network needs clip_feat"); return LION_ERR_ARG; }
  // any batch size: chunks of 32 shapes (the reference takes any B, resnet.py:195-218)
  for (int b0 = 0; b0 < B; b0 += GP_MAXB) {
    const int nb = B - b0 < GP_MAXB ? B - b0 : GP_MAXB;
    const size_t mk = c->mark();
    const float* xc = x + (size_t)b0 * g->D;
    const float* cc = clip ? clip + (size_t)b0 * g->clip_dim : nullptr;
    float* oc = out + (size_t)b0 * g->D;
    LION_TRY(global_prior_forward_layers(m, xc, t + b0, cc, oc, nb, rec, b0));
    c->release(mk);
  }
  return 0;
}

}  // namespace lion

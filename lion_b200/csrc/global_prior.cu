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
// mul: result *= mul[b][o] (SE gate, or the scaled dropout mask after conv1's ReLU);  res: result += res[b][o] (residual
// shortcut);  act_out: the activation before mul, [B][O] (the SE gate sigmoid(fc2) the training forward saves)
__global__ void k_gp_reduce(const float* __restrict__ part, int nsplit, const float* __restrict__ bias, float* __restrict__ out,
                            int out_stride, const float* __restrict__ mul, int mul_stride, const float* __restrict__ res,
                            int res_stride, int B, int O, int act, float* __restrict__ act_out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * O) return;
  int b = i / O, o = i % O;
  float v = 0.0f;
  for (int s = 0; s < nsplit; ++s) v += part[((size_t)s * B + b) * O + o];
  v += bias ? bias[o] : 0.0f;
  if (act == 1) v = fmaxf(v, 0.0f);
  else if (act == 2) v = 1.0f / (1.0f + expf(-v));
  if (act_out) act_out[(size_t)b * O + o] = v;
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

// The Linears' tensors in lion_params() order, taken from `cur`: the parameters at build, their gradients in a backward.
static void gp_bind(GlobalPriorBlk* g, Cursor& cur) {
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
}

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
  gp_bind(g, cur);
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
                     const float* mul, int ms, const float* res, int rs, int B, int act, float* act_out = nullptr) {
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
  LION_LAUNCH(c, k_gp_reduce, cdiv(B * l.O, 256), 256, 0, part, nsplit, l.b, out, os, mul, ms, res, rs, B, l.O, act, act_out);
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
// drop: the scaled dropout masks of this chunk's rows, cell k's at drop + k * drop_cell ([B][nf] each), or null
static int global_prior_forward_layers(Model* m, const float* x, const float* t, const float* clip, float* out, int B,
                                       const GpRecord* rec, int b0, const float* drop, size_t drop_cell) {
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
    // conv1(x + t [| clip]) -> ReLU -> dropout (the mask in the reduce's mul slot; none in eval) -> conv2 -> ReLU -> SE -> + x
    const float* dm = drop ? drop + k * drop_cell : nullptr;
    if (g->clip) {
      if (!c->dry)
        LION_CHECK_CUDA(cudaMemcpy2DAsync(cat, tw * sizeof(float), h, nf * sizeof(float), nf * sizeof(float), B, cudaMemcpyDeviceToDevice, c->stream));
      LION_TRY(gp_linear(c, cell.c1, cat, tw, tadd, tw, a, nf, dm, nf, nullptr, 0, B, 1));
    } else {
      LION_TRY(gp_linear(c, cell.c1, h, nf, tadd, tw, a, nf, dm, nf, nullptr, 0, B, 1));
    }
    LION_TRY(gp_tap(c, rc.a, b0, a, nf, nf, B));
    LION_TRY(gp_linear(c, cell.c2, a, nf, nullptr, 0, bb, nf, nullptr, 0, nullptr, 0, B, 1));
    LION_TRY(gp_tap(c, rc.bb, b0, bb, nf, nf, B));
    LION_TRY(gp_linear(c, cell.se0, bb, nf, nullptr, 0, s0, nf / 8, nullptr, 0, nullptr, 0, B, 1));
    LION_TRY(gp_tap(c, rc.s, b0, s0, nf / 8, nf / 8, B));
    LION_TRY(gp_linear(c, cell.se2, s0, nf / 8, nullptr, 0, h2, nf, bb, nf, h, nf, B, 2,     // sigmoid(.) * bb + h
                       rc.gate ? rc.gate + (size_t)b0 * nf : nullptr));
    LION_TRY(gp_tap(c, rc.h, b0, h2, nf, nf, B));
    float* tmp = h; h = h2; h2 = tmp;
  }
  LION_TRY(gp_linear(c, g->outl, h, nf, nullptr, 0, out, g->D, nullptr, 0, nullptr, 0, B, 0));
  return check_launch(c, "global_prior_forward");
}

int global_prior_forward(Model* m, const float* x, const float* t, const float* clip, float* out, int B, const GpRecord* rec,
                         const float* drop) {
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
    const float* dc = drop ? drop + (size_t)b0 * g->nf : nullptr;
    LION_TRY(global_prior_forward_layers(m, xc, t + b0, cc, oc, nb, rec, b0, dc, (size_t)B * g->nf));
    c->release(mk);
  }
  return 0;
}

// =====================================================================================================================
// Training: a forward that keeps what the backward reads, and the backward of the whole network.
// Reference: the autograd of Prior.forward (resnet.py:195-218) through ResBlockSEDrop / ResBlockSEClip and SE.
// =====================================================================================================================

// The saved-activation buffer, [B][width] fp32 tensors back to back (include/lion_b200.h): x [D], pe [emb], t0 [4 emb],
// temb [nf], cmap [nf] (CLIP only), h0 [nf], then per cell a [nf], bb [nf], s [nf/8], gate [nf], h [nf].
struct GpSaved {
  float *x, *pe, *t0, *temb, *cmap, *h0;
  std::vector<GpRecord::Cell> cells;
};
static size_t gp_saved_layout(const GlobalPriorBlk* g, float* base, int B, GpSaved* s) {
  size_t off = 0;
  auto take = [&](int w) { float* p = base ? base + off : nullptr; off += (size_t)B * w; return p; };
  GpSaved l;
  l.x = take(g->D); l.pe = take(g->emb); l.t0 = take(g->emb * 4); l.temb = take(g->nf);
  l.cmap = g->clip ? take(g->nf) : nullptr;
  l.h0 = take(g->nf);
  l.cells.resize(g->ncell);
  for (auto& c : l.cells) { c.a = take(g->nf); c.bb = take(g->nf); c.s = take(g->nf / 8); c.gate = take(g->nf); c.h = take(g->nf); }
  if (s) *s = l;
  return off;
}
size_t global_prior_saved_floats(const Model* m, int B) { return gp_saved_layout(m->gp, nullptr, B, nullptr); }

// The forward of lion_global_prior_forward (the same launches, so the same bits) with the dropout masks applied and the
// activations the backward reads recorded into `saved`.
int global_prior_forward_train(Model* m, const float* x, const float* t, const float* clip, const float* drop,
                               float* saved, float* out, int B) {
  GlobalPriorBlk* g = m->gp;
  GpSaved s;
  gp_saved_layout(g, saved, B, &s);
  LION_TRY(memcpy_d2d(m->ctx, s.x, x, sizeof(float) * B * g->D));
  GpRecord rec;
  rec.pe = s.pe; rec.t0 = s.t0; rec.temb = s.temb; rec.cmap = s.cmap; rec.h0 = s.h0;
  rec.cells = s.cells.data();
  return global_prior_forward(m, x, t, clip, out, B, &rec, drop);
}

// dgrad, phase 1:  part[os][b][k] = sum_{o in slice os} g~[b][o] * W~[o][k]
// grid = (K/128, O/256, B/32).  The weight tile [256 o x 128 k] (128 KB) is read k-contiguous, as it lies in memory, and
// streams in four 64-row cp.async commit groups like k_gp_partial's; mma.sync.m16n8k8 TF32 with M = 16 columns k of W
// per warp (A[m][o] = W[o][k], a transposed read of the row-major tile), N = 8 shapes, the MMA's K = o.
// Operand model, the forward's: the gradient g is staged through registers and rounded with cvt.rna (an unbiased
// rounding, as for the forward's activations); the weights go HBM -> shared memory by cp.async unrounded and reach the
// tensor core as fp32 bits, which it reads truncated to TF32 -- rounding them would cost a register pass over every
// weight tile, and truncation of the weights is what the forward applied to them too.
// Pitches: W 136 floats (bank = 8 o + k across a fragment), g 260 (bank = 4 b + o): no bank conflicts.
// Deterministic: the o slices are summed in a fixed order by k_gpb_reduce.
constexpr int GB_KT = 128;      // W columns (outputs of the dgrad) per block
constexpr int GB_OS = 256;      // W rows (the reduction) per block
constexpr int GB_WP = GB_KT + 8;
constexpr int GB_GP = GB_OS + 4;
constexpr int GB_MAXSPLIT = 16;
__global__ void __launch_bounds__(GP_WARPS * 32, 1)
k_gpb_dgrad(const float* __restrict__ W, const float* __restrict__ g, int gs, float* __restrict__ part, int B, int K, int O) {
  extern __shared__ __align__(16) float s_mem[];
  float* s_w = s_mem;                          // [GB_OS][GB_WP]
  float* s_g = s_mem + GB_OS * GB_WP;          // [GP_BT][GB_GP]
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int k0 = blockIdx.x * GB_KT, kt = min(GB_KT, K - k0);
  const int o0 = blockIdx.y * GB_OS;
  const int b0 = blockIdx.z * GP_BT;
  const uint32_t s_w_addr = (uint32_t)__cvta_generic_to_shared(s_w);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
#pragma unroll
    for (int u = 0; u < (64 * GB_KT / 4) / (GP_WARPS * 32); ++u) {    // 64 rows x 32 pieces / 256 threads = 8
      int c = tid + u * (GP_WARPS * 32);
      int row = q * 64 + (c >> 5), col = (c & 31) * 4;
      if (o0 + row < O && col < kt)
        cp_async16(s_w_addr + (uint32_t)(row * GB_WP + col) * 4u, W + (size_t)(o0 + row) * K + k0 + col);
      else   // rows past O meet zero gradients; columns past K are never stored
        *reinterpret_cast<float4*>(s_w + row * GB_WP + col) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  {
    constexpr int PER_THREAD = GP_BT * (GB_OS / 4) / (GP_WARPS * 32);      // 8
#pragma unroll
    for (int u = 0; u < PER_THREAD; ++u) {
      int i = tid + u * (GP_WARPS * 32);
      int b = i / (GB_OS / 4), o = (i % (GB_OS / 4)) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b0 + b < B && o0 + o < O) v = *reinterpret_cast<const float4*>(g + (size_t)(b0 + b) * gs + o0 + o);
      *reinterpret_cast<float4*>(s_g + b * GB_GP + o) = make_float4(
          __uint_as_float(tf32_bits(v.x)), __uint_as_float(tf32_bits(v.y)), __uint_as_float(tf32_bits(v.z)), __uint_as_float(tf32_bits(v.w)));
    }
  }
  const int g8 = lane >> 2, t4 = lane & 3;
  float acc[4][4];
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[n][i] = 0.0f;
  const float* wa = s_w + t4 * GB_WP + wid * 16 + g8;      // A(m = g8, o = t4) of this warp's 16 columns
  const float* gb = s_g + g8 * GB_GP + t4;                  // B(o = t4, shape g8) of each 8-shape tile
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (q == 0) asm volatile("cp.async.wait_group 3;" ::: "memory");
    else if (q == 1) asm volatile("cp.async.wait_group 2;" ::: "memory");
    else if (q == 2) asm volatile("cp.async.wait_group 1;" ::: "memory");
    else asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    if (o0 + q * 64 < O) {
#pragma unroll
      for (int kk = 0; kk < 64; kk += 8) {
        const int o = q * 64 + kk;
        uint32_t a0 = __float_as_uint(wa[o * GB_WP]), a1 = __float_as_uint(wa[o * GB_WP + 8]);
        uint32_t a2 = __float_as_uint(wa[(o + 4) * GB_WP]), a3 = __float_as_uint(wa[(o + 4) * GB_WP + 8]);
#pragma unroll
        for (int n = 0; n < 4; ++n) {
          uint32_t v0 = __float_as_uint(gb[n * 8 * GB_GP + o]), v1 = __float_as_uint(gb[n * 8 * GB_GP + o + 4]);
          asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                       : "+f"(acc[n][0]), "+f"(acc[n][1]), "+f"(acc[n][2]), "+f"(acc[n][3])
                       : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(v0), "r"(v1));
        }
      }
    }
  }
  float* pout = part + (size_t)blockIdx.y * B * K;
#pragma unroll
  for (int n = 0; n < 4; ++n) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      int k = k0 + wid * 16 + g8 + (i >= 2 ? 8 : 0);
      int b = b0 + n * 8 + 2 * t4 + (i & 1);
      if (b < B && k < K) pout[(size_t)b * K + k] = acc[n][i];
    }
  }
}

// dgrad, phase 2: v = sum_os part[os][b][k], then the elementwise backward that sits between this Linear and the next
// one back.  Columns k < split ([B][split] arrays, row stride split) in this order:
//   v += add_a * add_b        (the SE product's direct term d/d bb = g_h * gate, at fc0's input)
//   v  = relu > 0 ? v : 0     (ReLU, from the saved post-activation; after dropout a kept value is > 0 iff its input was)
//   v *= mul                  (the scaled dropout mask)
//   acc = [acc +] v           (the sum over cells of d/d temb; acc_add = 0 for the first cell summed)
//   out = v [+ res]           (the residual fan-out: d/d h_in = d/d h_out + d/d (h_in + temb))
//   gz  = out * bb * gate * (1 - gate)   (the previous cell's d/d fc2 pre-sigmoid, from its d/d h_out)
// Columns k >= split (the CLIP half of conv1's input): acc2 = [acc2 +] v.
struct GbEpi {
  int split = 0;
  float* out = nullptr;
  const float *add_a = nullptr, *add_b = nullptr, *relu = nullptr, *mul = nullptr, *res = nullptr;
  float* acc = nullptr; float* acc2 = nullptr; int acc_add = 0;
  const float *se_bb = nullptr, *se_gate = nullptr; float* gz = nullptr;
};
__global__ void k_gpb_reduce(const float* __restrict__ part, int nsplit, int B, int K, GbEpi e) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  int b = i / K, k = i % K;
  float v = 0.0f;
  for (int s = 0; s < nsplit; ++s) v += part[((size_t)s * B + b) * K + k];
  if (k >= e.split) {
    const size_t j = (size_t)b * (K - e.split) + k - e.split;
    e.acc2[j] = e.acc_add ? e.acc2[j] + v : v;
    return;
  }
  const size_t j = (size_t)b * e.split + k;
  if (e.add_a) v = fmaf(e.add_a[j], e.add_b[j], v);
  if (e.relu) v = e.relu[j] > 0.0f ? v : 0.0f;
  if (e.mul) v *= e.mul[j];
  if (e.acc) e.acc[j] = e.acc_add ? e.acc[j] + v : v;
  if (e.res) v += e.res[j];
  e.out[j] = v;
  if (e.gz) {
    const float s = e.se_gate[j];
    e.gz[j] = v * e.se_bb[j] * (s * (1.0f - s));
  }
}

// wgrad:  dW[o][k] = sum_b g[b][o] * x~[b][k],  db[o] = sum_b g[b][o],  b = 0 .. B-1 in order, all shapes in one pass.
// Operand model: x~ is the operand the forward's k_gp_partial consumed, cvt.rna of fl32(x + add) (for the CLIP conv1,
// columns >= split come from x2: [h + temb | cmap]); g is the fp32 gradient, not rounded.  The products and sums are
// fp32 FFMA: with B <= 64 shapes as the K of this GEMM, the 2 B flops per weight are cheap next to writing the weight
// gradient, so the tensor cores would save nothing and TF32 rounding of g would cost 2^-11 of accuracy.
// grid = (K/128, O/32); thread (tk = lane, to = warp) owns a 4 x 4 block dW[o0 + 4 to ..][k0 + 4 tk ..], stored as float4.
constexpr int GW_KT = 128, GW_OT = 32, GW_BT = 32;
__global__ void __launch_bounds__(256)
k_gpb_wgrad(const float* __restrict__ g, int gs, const float* __restrict__ x, int xs, const float* __restrict__ add, int as,
            const float* __restrict__ x2, int x2s, int split, float* __restrict__ dW, float* __restrict__ db, int B, int K, int O) {
  __shared__ __align__(16) float s_x[GW_BT][GW_KT];
  __shared__ __align__(16) float s_g[GW_BT][GW_OT];
  const int tid = threadIdx.x, tk = tid & 31, to = tid >> 5;
  const int k0 = blockIdx.x * GW_KT, o0 = blockIdx.y * GW_OT;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int b0 = 0; b0 < B; b0 += GW_BT) {
    __syncthreads();
#pragma unroll
    for (int u = 0; u < GW_BT * (GW_KT / 4) / 256; ++u) {      // 4
      int i = tid + u * 256;
      int b = i >> 5, k = k0 + (i & 31) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b0 + b < B && k < K) {
        if (k < split) {
          v = *reinterpret_cast<const float4*>(x + (size_t)(b0 + b) * xs + k);
          if (add) {
            float4 a = *reinterpret_cast<const float4*>(add + (size_t)(b0 + b) * as + k);
            v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
          }
        } else {
          v = *reinterpret_cast<const float4*>(x2 + (size_t)(b0 + b) * x2s + k - split);
        }
      }
      *reinterpret_cast<float4*>(&s_x[b][(i & 31) * 4]) = f4_tf32(v);
    }
#pragma unroll
    for (int u = 0; u < GW_BT * GW_OT / 256; ++u) {            // 4
      int i = tid + u * 256;
      int b = i >> 5, o = i & 31;
      s_g[b][o] = (b0 + b < B && o0 + o < O) ? g[(size_t)(b0 + b) * gs + o0 + o] : 0.0f;
    }
    __syncthreads();
    const int nb = min(GW_BT, B - b0);
    for (int b = 0; b < nb; ++b) {
      float4 xv = *reinterpret_cast<const float4*>(&s_x[b][tk * 4]);
      float4 gv = *reinterpret_cast<const float4*>(&s_g[b][to * 4]);
      const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[i][0] = fmaf(gg[i], xv.x, acc[i][0]); acc[i][1] = fmaf(gg[i], xv.y, acc[i][1]);
        acc[i][2] = fmaf(gg[i], xv.z, acc[i][2]); acc[i][3] = fmaf(gg[i], xv.w, acc[i][3]);
      }
    }
  }
  const int k = k0 + tk * 4;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int o = o0 + to * 4 + i;
    if (o < O && k < K) *reinterpret_cast<float4*>(dW + (size_t)o * K + k) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  }
  if (db && blockIdx.x == 0 && tk < 4) {
    const int o = o0 + to * 4 + tk;
    if (o < O) {
      float v = 0.0f;
      for (int b = 0; b < B; ++b) v += g[(size_t)b * gs + o];
      db[o] = v;
    }
  }
}

// dx = g W for all B rows (chunks of 32 on grid.z) through the epilogue e (e.split = l.K unless it is the CLIP conv1)
static int gpb_dgrad(Ctx* c, const GPLin& l, const float* g, int gs, int B, const GbEpi& e) {
  if (l.K % 4 || l.O % 4) {
    set_error("global prior backward: K=%d and O=%d must be multiples of 4 (16-byte loads)", l.K, l.O);
    return LION_ERR_ARG;
  }
  const int nsplit = cdiv(l.O, GB_OS);
  if (nsplit > GB_MAXSPLIT) {
    set_error("global prior backward: O=%d needs %d slices of %d, at most %d", l.O, nsplit, GB_OS, GB_MAXSPLIT);
    return LION_ERR_ARG;
  }
  const size_t smem = (size_t)(GB_OS * GB_WP + GP_BT * GB_GP) * sizeof(float);
  static DevOnce attr_once;
  if (attr_once.need()) LION_CHECK_CUDA(cudaFuncSetAttribute(k_gpb_dgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  size_t mk = c->mark();
  float* part = c->alloc_n<float>((size_t)nsplit * B * l.K);
  LION_LAUNCH(c, k_gpb_dgrad, dim3(cdiv(l.K, GB_KT), nsplit, cdiv(B, GP_BT)), GP_WARPS * 32, smem, l.w, g, gs, part, B, l.K, l.O);
  LION_LAUNCH(c, k_gpb_reduce, cdiv(B * l.K, 256), 256, 0, part, nsplit, B, l.K, e);
  c->release(mk);
  return 0;
}

// dW, db of Linear l (gl: its gradient tensors) from the gradient g at its output and its forward operand
static int gpb_wgrad(Ctx* c, const GPLin& gl, const float* g, int gs, const float* x, int xs, const float* add, int as,
                     int B, const float* x2 = nullptr, int x2s = 0, int split = -1) {
  // gl.w / gl.b point into the caller's gradient buffers, bound through the parameter Cursor (const there)
  LION_LAUNCH(c, k_gpb_wgrad, dim3(cdiv(gl.K, GW_KT), cdiv(gl.O, GW_OT)), 256, 0, g, gs, x, xs, add, as, x2, x2s,
              split < 0 ? gl.K : split, const_cast<float*>(gl.w), const_cast<float*>(gl.b), B, gl.K, gl.O);
  return 0;
}

int global_prior_backward(Model* m, const float* saved, const float* clip, const float* drop, const float* gout,
                          float* gx, const float* const* gparams, int nparams, int B, const GpBwdRecord* rec) {
  const GlobalPriorBlk* g = m->gp;
  Ctx* c = m->ctx;
  if (g->clip && !clip) { set_error("global prior backward: this network needs clip_feat"); return LION_ERR_ARG; }
  GlobalPriorBlk gg;          // the same Linears, w / b pointing at the gradients
  gg.D = g->D; gg.nf = g->nf; gg.emb = g->emb; gg.ncell = g->ncell; gg.clip = g->clip; gg.clip_dim = g->clip_dim;
  Cursor cur{gparams, nparams};
  gp_bind(&gg, cur);
  if (cur.bad || cur.i != cur.n) {
    set_error("global prior backward: %d parameter gradients given, %d expected", nparams, (int)m->params.size());
    return LION_ERR_ARG;
  }
  GpSaved s;
  gp_saved_layout(g, const_cast<float*>(saved), B, &s);
  const int nf = g->nf, D = g->D, E4 = g->emb * 4, nc = g->ncell;
  float* gh = c->alloc_n<float>((size_t)B * nf);       // d/d (cell output), then d/d (cell input) in place
  float* gz = c->alloc_n<float>((size_t)B * nf);
  float* gsq = c->alloc_n<float>((size_t)B * nf / 8);
  float* gbb = c->alloc_n<float>((size_t)B * nf);
  float* gz1 = c->alloc_n<float>((size_t)B * nf);
  float* gtemb = c->alloc_n<float>((size_t)B * nf);
  float* gcmap = g->clip ? c->alloc_n<float>((size_t)B * nf) : nullptr;
  float* gt0 = c->alloc_n<float>((size_t)B * E4);
  const GpBwdRecord no_rec;
  const GpBwdRecord& r = rec ? *rec : no_rec;

  // output layer; its dgrad epilogue starts the last cell's SE backward
  const GpRecord::Cell& last = s.cells[nc - 1];
  LION_TRY(gpb_wgrad(c, gg.outl, gout, D, last.h, nf, nullptr, 0, B));
  GbEpi e;
  e.split = nf; e.out = gh; e.se_bb = last.bb; e.se_gate = last.gate; e.gz = gz;
  LION_TRY(gpb_dgrad(c, g->outl, gout, D, B, e));
  for (int k = nc - 1; k >= 0; --k) {
    const auto& cell = g->cells[k];
    const auto& gc = gg.cells[k];
    const GpRecord::Cell& sc = s.cells[k];
    const float* h_in = k ? s.cells[k - 1].h : s.h0;
    const GpBwdRecord::Cell rc = r.cells ? r.cells[k] : GpBwdRecord::Cell{};
    LION_TRY(gp_tap(c, rc.gh, 0, gh, nf, nf, B));
    LION_TRY(gp_tap(c, rc.gz, 0, gz, nf, nf, B));
    // SE fc.2: z = W2 s; gate = sigmoid(z)
    LION_TRY(gpb_wgrad(c, gc.se2, gz, nf, sc.s, nf / 8, nullptr, 0, B));
    e = GbEpi{}; e.split = nf / 8; e.out = gsq; e.relu = sc.s;
    LION_TRY(gpb_dgrad(c, cell.se2, gz, nf, B, e));
    LION_TRY(gp_tap(c, rc.gs, 0, gsq, nf / 8, nf / 8, B));
    // SE fc.0: s = relu(W1 bb); bb also reaches the output directly through bb * gate
    LION_TRY(gpb_wgrad(c, gc.se0, gsq, nf / 8, sc.bb, nf, nullptr, 0, B));
    e = GbEpi{}; e.split = nf; e.out = gbb; e.add_a = gh; e.add_b = sc.gate; e.relu = sc.bb;
    LION_TRY(gpb_dgrad(c, cell.se0, gsq, nf / 8, B, e));
    LION_TRY(gp_tap(c, rc.gbb, 0, gbb, nf, nf, B));
    // conv2: bb = relu(W a + b), a = dropout(relu(conv1))
    LION_TRY(gpb_wgrad(c, gc.c2, gbb, nf, sc.a, nf, nullptr, 0, B));
    e = GbEpi{}; e.split = nf; e.out = gz1; e.relu = sc.a; e.mul = drop ? drop + (size_t)k * B * nf : nullptr;
    LION_TRY(gpb_dgrad(c, cell.c2, gbb, nf, B, e));
    LION_TRY(gp_tap(c, rc.gz1, 0, gz1, nf, nf, B));
    // conv1 on [h_in + temb | cmap]: the residual, the temb sum and the CLIP half; then the previous cell's SE gate
    LION_TRY(gpb_wgrad(c, gc.c1, gz1, nf, h_in, nf, s.temb, nf, B, s.cmap, nf, nf));
    e = GbEpi{}; e.split = nf; e.out = gh; e.res = gh; e.acc = gtemb; e.acc2 = gcmap; e.acc_add = k < nc - 1;
    if (k > 0) { e.se_bb = s.cells[k - 1].bb; e.se_gate = s.cells[k - 1].gate; e.gz = gz; }
    LION_TRY(gpb_dgrad(c, cell.c1, gz1, nf, B, e));
  }
  LION_TRY(gp_tap(c, r.gh0, 0, gh, nf, nf, B));
  LION_TRY(gp_tap(c, r.gtemb, 0, gtemb, nf, nf, B));
  if (g->clip) LION_TRY(gp_tap(c, r.gcmap, 0, gcmap, nf, nf, B));
  // input layer -> dx
  LION_TRY(gpb_wgrad(c, gg.in, gh, nf, s.x, D, nullptr, 0, B));
  e = GbEpi{}; e.split = D; e.out = gx;
  LION_TRY(gpb_dgrad(c, g->in, gh, nf, B, e));
  // time embedding (no gradient reaches t) and clip_feat_mapping (none reaches clip_feat)
  LION_TRY(gpb_wgrad(c, gg.t1, gtemb, nf, s.t0, E4, nullptr, 0, B));
  e = GbEpi{}; e.split = E4; e.out = gt0;
  LION_TRY(gpb_dgrad(c, g->t1, gtemb, nf, B, e));
  LION_TRY(gp_tap(c, r.gt0, 0, gt0, E4, E4, B));
  LION_TRY(gpb_wgrad(c, gg.t0, gt0, E4, s.pe, g->emb, nullptr, 0, B));
  if (g->clip) LION_TRY(gpb_wgrad(c, gg.cmap, gcmap, nf, clip, g->clip_dim, nullptr, 0, B));
  return check_launch(c, "global_prior_backward");
}

}  // namespace lion

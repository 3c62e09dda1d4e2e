// lion_b200 -- host orchestration of the PVCNN2-AdaGN U-Net and its blocks on the packed
// layouts of packed_kernels.cuh, plus the network/block C ABI.
//
// Reference being replaced (paths relative to the reference repository):
//   models/latent_points_ada.py:117-173      PVCNN2Unet.forward
//   models/pvcnn2_ada.py:235-280             PVConv.forward
//   models/pvcnn2_ada.py:354-382, :98-114    PointNetSAModule.forward, BallQuery.forward
//   models/pvcnn2_ada.py:393-411             PointNetFPModule.forward
//   models/pvcnn2_ada.py:54-71               LinearAttention.forward
//   models/pvcnn2_ada.py:140-164             SharedMLP.forward
//   models/adagn.py:45-65                    AdaGN.forward
// What is restructured relative to the reference (same arithmetic, fewer passes):
//   * the 61 AdaGN style Linears run as ONE kernel per forward (style is step-invariant);
//   * GroupNorm statistics come out of the producing convolution's epilogue; GroupNorm,
//     the style affine and (after the 2nd conv) the SE gate fold into one per-(b,c) affine
//     that the next consumer applies on load (activation pass / devoxelisation);
//   * voxel indices, counts and normalised coordinates are computed once per distinct
//     (coords, resolution) -- 4x per step instead of 14x;
//   * no permutes: the latent [B,N,4] is already a packed-feature tensor.
#include <algorithm>
#include <deque>
#include <memory>
#include <cstdlib>
#include <cmath>
#include "common.cuh"
#include "packed_kernels.cuh"
#include "model.cuh"
#include "../../include/lion_b200.h"

namespace lion {

// =====================================================================================
// error state, context
// =====================================================================================
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

int ctx_reserve(Ctx* c, size_t bytes) {
  if (bytes <= c->cap) return 0;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(c->stream, &st);
  if (st != cudaStreamCaptureStatusNone) {
    set_error("scratch arena too small (%zu > %zu bytes) during stream capture: run one eager warm-up call first", bytes, c->cap);
    return LION_ERR_STATE;
  }
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  if (c->base) LION_CHECK_CUDA(cudaFree(c->base));
  c->base = nullptr;
  c->cap = 0;
  size_t want = bytes + bytes / 8 + (size_t(1) << 20);
  cudaError_t e = cudaMalloc((void**)&c->base, want);
  if (e != cudaSuccess) {
    set_error("cudaMalloc(%zu) for the scratch arena failed: %s", want, cudaGetErrorString(e));
    return LION_ERR_OOM;
  }
  c->cap = want;
  c->generation++;           // every CUDA graph captured on this context so far has the old addresses baked in
  return 0;
}

// persistent zero grid: (re)allocated and zeroed outside graph capture; users keep it all-zero
int ctx_reserve_zgrid(Ctx* c, size_t bytes) {
  if (bytes <= c->zgrid_cap) return 0;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(c->stream, &st);
  if (st != cudaStreamCaptureStatusNone) {
    set_error("zero grid too small during stream capture: run one eager warm-up call first");
    return LION_ERR_STATE;
  }
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  if (c->zgrid) LION_CHECK_CUDA(cudaFree(c->zgrid));
  c->zgrid = nullptr; c->zgrid_cap = 0;
  cudaError_t e = cudaMalloc((void**)&c->zgrid, bytes);
  if (e != cudaSuccess) { set_error("cudaMalloc(%zu) for the zero grid failed: %s", bytes, cudaGetErrorString(e)); return LION_ERR_OOM; }
  LION_CHECK_CUDA(cudaMemset(c->zgrid, 0, bytes));
  c->zgrid_cap = bytes;
  c->generation++;
  return 0;
}

// weight packing kernels
__global__ void k_pack_conv_w(const float* __restrict__ w_src, const int* __restrict__ kmap, float* __restrict__ wt,
                              int ntaps, int cin_ref, int cin_pad, int cout, int cout_pad) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t total = (size_t)ntaps * cin_pad * cout_pad;
  if (i >= total) return;
  int co = i % cout_pad;
  int ci = (i / cout_pad) % cin_pad;
  int t = i / ((size_t)cout_pad * cin_pad);
  int src = kmap[ci];
  float v = 0.0f;
  if (src >= 0 && co < cout) v = w_src[((size_t)co * cin_ref + src) * ntaps + t];
  wt[i] = v;
}
// sparse first convolution: the 27 taps side by side, wy[ci][t * cout_pad + co] = wt[t][ci][co] (zero beyond 27 * cout_pad)
__global__ void k_pack_taps_wide(const float* __restrict__ wt, float* __restrict__ wy, int cin_pad, int cout_pad, int ny_pad) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)cin_pad * ny_pad) return;
  int n = i % ny_pad, ci = i / ny_pad;
  int t = n / cout_pad, co = n % cout_pad;
  wy[i] = t < 27 ? wt[((size_t)t * cin_pad + ci) * cout_pad + co] : 0.0f;
}
__global__ void k_pad_vec(const float* __restrict__ src, float* __restrict__ dst, int n, int n_pad) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_pad) dst[i] = i < n ? src[i] : 0.0f;
}


// build a conv's packed forms. kmap: packed input channel -> reference input channel (-1 = zero)
int make_conv(Model* m, ConvW& w, const float* w_src, const float* b_src, int ntaps, int cin_ref, int cout,
              const std::vector<int>& kmap) {
  w.ntaps = ntaps; w.cin_ref = cin_ref; w.cin_pad = (int)kmap.size(); w.cout = cout;
  w.cout_pad = (cout <= 4) ? 4 : roundup(cout, 8);
  if (!w_src) { set_error("model parameters exhausted while building a convolution"); return LION_ERR_ARG; }
  if (w.cin_pad % 4) { set_error("packed input channels must be a multiple of 4 (got %d)", w.cin_pad); return LION_ERR_ARG; }
  int* kmap_dev = nullptr;
  LION_TRY(m->dmalloc(&kmap_dev, kmap.size()));
  LION_CHECK_CUDA(cudaMemcpy(kmap_dev, kmap.data(), kmap.size() * sizeof(int), cudaMemcpyHostToDevice));
  const size_t nw = (size_t)ntaps * w.cin_pad * w.cout_pad;
  LION_TRY(m->dmalloc(&w.wt, nw));
  m->repack.push_back([w_src, kmap_dev, wt = w.wt, ntaps, cin_ref, cin_pad = w.cin_pad, cout, cout_pad = w.cout_pad, nw] {
    k_pack_conv_w<<<(unsigned)cdivz(nw, 256), 256>>>(w_src, kmap_dev, wt, ntaps, cin_ref, cin_pad, cout, cout_pad);
  });
  if (b_src) {
    LION_TRY(m->dmalloc(&w.bias, (size_t)w.cout_pad));
    m->repack.push_back([b_src, bias = w.bias, cout, cout_pad = w.cout_pad] {
      k_pad_vec<<<cdiv(cout_pad, 128), 128>>>(b_src, bias, cout, cout_pad);
    });
  }
  LION_TRY(conv_tc_prepare(m, w));     // optional tensor-core packing (adds its own step)
  return 0;
}
std::vector<int> ident_map(int c) {
  std::vector<int> k(roundup(c, 4), -1);
  for (int i = 0; i < c; ++i) k[i] = i;
  return k;
}

int run_repack(Model* m) {
  for (auto& step : m->repack) step();
  LION_CHECK_CUDA(cudaGetLastError());
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  return 0;
}

// The FP16 packings of the convolutions an FP16 forward uses (the second convolution of every PVConv, or a stand-alone
// Conv3d), made on the model's first FP16 forward: allocated, packed now, and re-packed by lion_model_refresh with the
// TF32 ones.  Allocation is not capturable: the first FP16 call must be eager (the samplers' first step is).
static int ensure_f16(Model* m, void* stream) {
  // the context's mutex: the first FP16 calls of two threads, or one and a lion_model_refresh, must not both append to
  // m->repack or pack tc16
  std::unique_lock<std::mutex> lock;
  if (m->ctx->mu) lock = std::unique_lock<std::mutex>(*m->ctx->mu);
  if (m->f16_ready) return 0;
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing((cudaStream_t)stream, &st);
  LION_REQUIRE(st == cudaStreamCaptureStatusNone, "FP16 forward: the model's first FP16 call must run outside stream capture");
  LION_CHECK_CUDA(cudaSetDevice(m->ctx->device));
  const size_t first = m->repack.size();
  auto pv = [&](std::vector<std::vector<Block>>& levels) -> int {
    for (auto& lv : levels) for (auto& b : lv) if (b.kind == LION_KIND_PVCONV) LION_TRY(conv_tc_prepare_f16(m, b.pv.c2));
    return 0;
  };
  if (m->unet) { LION_TRY(pv(m->unet->sa)); LION_TRY(pv(m->unet->fp)); }
  if (m->block && m->block->kind == LION_KIND_PVCONV) LION_TRY(conv_tc_prepare_f16(m, m->block->pv.c2));
  if (m->kind == LION_KIND_CONV3D) LION_TRY(conv_tc_prepare_f16(m, m->conv_single));
  for (size_t i = first; i < m->repack.size(); ++i) m->repack[i]();
  LION_CHECK_CUDA(cudaGetLastError());
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  m->f16_ready = true;
  return 0;
}

// plain: nn.GroupNorm(8, C) of the non-Ada blocks (models/pvcnn2.py) = AdaGN whose style Linear is identically
// (factor, bias) = (1, 0): no `emd` parameters are consumed and k_style_linear writes the constants.
int make_adagn(Model* m, AdaGNW& g, Cursor& cur, int C, bool plain = false) {
  g.C = C;
  g.gamma = cur.next(); g.beta = cur.next();
  const float* ew = plain ? nullptr : cur.next(); const float* eb = plain ? nullptr : cur.next();
  if (cur.bad) { set_error("model parameters exhausted while building AdaGN(%d)", C); return LION_ERR_ARG; }
  if (C % 8 || C > 512) { set_error("AdaGN channels must be a multiple of 8 and <= 512 (got %d)", C); return LION_ERR_ARG; }
  g.style_off = m->style_total;
  m->style_layers.push_back({ew, eb, 2 * C, m->style_total});
  m->style_total += 2 * C;
  return 0;
}

// SharedMLP: n x (1x1 conv, AdaGN, Swish); first conv's input mapping is given
int make_shared_mlp(Model* m, SharedMLPBlk& b, Cursor& cur, int cin_ref, const std::vector<int>& kmap0,
                    const std::vector<int>& outs, bool plain = false) {
  int cin = cin_ref;
  b.cin_pad = (int)kmap0.size();
  b.conv.resize(outs.size());
  b.gn.resize(outs.size());
  for (size_t i = 0; i < outs.size(); ++i) {
    const float* w = cur.next(); const float* bi = cur.next();
    if (cur.bad) { set_error("model parameters exhausted in SharedMLP"); return LION_ERR_ARG; }
    LION_TRY(make_conv(m, b.conv[i], w, bi, 1, cin, outs[i], i == 0 ? kmap0 : ident_map(cin)));
    LION_TRY(make_adagn(m, b.gn[i], cur, outs[i], plain));
    cin = outs[i];
  }
  return 0;
}
int make_attn(Model* m, AttnBlk& a, Cursor& cur, int C, int heads) {
  a.C = C; a.heads = heads;
  int hid = heads * 32;
  const float* qw = cur.next(); const float* ow = cur.next(); const float* ob = cur.next();
  if (cur.bad) { set_error("model parameters exhausted in LinearAttention"); return LION_ERR_ARG; }
  LION_TRY(make_conv(m, a.qkv, qw, nullptr, 1, C, 3 * hid, ident_map(C)));
  LION_TRY(make_conv(m, a.out, ow, ob, 1, hid, C, ident_map(hid)));
  return 0;
}
// cin need not be a multiple of 4: the input PF is padded to whole groups and the padding meets zero weights
int make_pvconv(Model* m, PVConvBlk& p, Cursor& cur, int cin, int cout, int r, bool attn, bool plain = false) {
  p.cin = roundup(cin, 4); p.cout = cout; p.r = r; p.has_attn = attn;
  const float* w1 = cur.next(); const float* b1 = cur.next();
  if (cur.bad) { set_error("model parameters exhausted in PVConv"); return LION_ERR_ARG; }
  LION_TRY(make_conv(m, p.c1, w1, b1, 27, cin, cout, ident_map(cin)));
  if ((p.c1.cout_pad == 32 || p.c1.cout_pad == 64) && p.c1.cout == p.c1.cout_pad && p.c1.cin_pad >= 16) {
    // weights of the sparse form of this convolution (pvconv_fwd): one GEMM x[v] -> y[v][27 taps][cout]
    ConvW& y = p.c1y;
    y.ntaps = 1; y.cin_ref = p.c1.cin_pad; y.cin_pad = p.c1.cin_pad;
    y.cout = y.cout_pad = roundup(27 * p.c1.cout_pad, 128);
    LION_TRY(m->dmalloc(&y.wt, (size_t)y.cin_pad * y.cout_pad));
    m->repack.push_back([wt = p.c1.wt, wy = y.wt, cin_pad = y.cin_pad, cout_pad = p.c1.cout_pad, ny_pad = y.cout_pad] {
      k_pack_taps_wide<<<(unsigned)cdivz((size_t)cin_pad * ny_pad, 256), 256>>>(wt, wy, cin_pad, cout_pad, ny_pad);
    });
    LION_TRY(conv_tc_prepare(m, y));     // packs y.wt: its step must follow the one above
  }
  LION_TRY(make_adagn(m, p.g1, cur, cout, plain));
  const float* w2 = cur.next(); const float* b2 = cur.next();
  if (cur.bad) { set_error("model parameters exhausted in PVConv"); return LION_ERR_ARG; }
  LION_TRY(make_conv(m, p.c2, w2, b2, 27, cout, cout, ident_map(cout)));
  LION_TRY(make_adagn(m, p.g2, cur, cout, plain));
  p.se1 = cur.next(); p.se2 = cur.next();
  // state_dict order of the reference PVConv: voxel_layers, attn, point_features (pvcnn2_ada.py:227-233)
  if (attn) LION_TRY(make_attn(m, p.attn, cur, cout, 4));
  LION_TRY(make_shared_mlp(m, p.point, cur, cin, ident_map(cin), {cout}, plain));
  if (cur.bad) { set_error("model parameters exhausted in PVConv"); return LION_ERR_ARG; }
  return 0;
}
int make_sa(Model* m, SABlk& s, Cursor& cur, int cfeat, int mcent, float radius, int k, const std::vector<int>& outs, bool plain = false) {
  s.cfeat = cfeat; s.m = mcent; s.radius = radius; s.k = k;
  if (cfeat % 4) { set_error("SA feature channels must be a multiple of 4 (got %d)", cfeat); return LION_ERR_ARG; }
  if (k != 32) { set_error("SA module: num_neighbors must be 32 (got %d)", k); return LION_ERR_ARG; }
  // reference input order: [rel-xyz(3) | features]  (pvcnn2_ada.py:113) -> packed [xyz,0 | features]
  std::vector<int> kmap(4 + cfeat, -1);
  kmap[0] = 0; kmap[1] = 1; kmap[2] = 2;
  for (int i = 0; i < cfeat; ++i) kmap[4 + i] = 3 + i;
  return make_shared_mlp(m, s.mlp, cur, cfeat + 3, kmap, outs, plain);
}
int make_fp(Model* m, FPBlk& f, Cursor& cur, int cc, int cp, const std::vector<int>& outs) {
  f.cc = cc; f.cp = cp;
  if (cc % 4) { set_error("FP interpolated channels must be a multiple of 4 (got %d)", cc); return LION_ERR_ARG; }
  // reference input order: [interpolated(cc) | skip(cp)] (pvcnn2_ada.py:402-406); skip padded to a group boundary
  std::vector<int> kmap(cc + roundup(cp, 4), -1);
  for (int i = 0; i < cc + cp; ++i) kmap[i] = i;
  return make_shared_mlp(m, f.mlp, cur, cc + cp, kmap, outs);
}

// =====================================================================================
// forward-time helpers
// =====================================================================================
struct PF { float4* p = nullptr; int G = 0; int R = 0; };
struct VoxPrep { const float4* c4; int N, r; float4* nc; int* order; int* ppos; int* len; unsigned char* occ; int occ_stride;
                 int* cidx; int* nocc; int* vgrid; };   // compact ids of the occupied voxels (sparse first convolution) or null
// Intermediate results of one MLP (an SA module's, an FP module's or the U-Net head's) that lion_sa_mlp_probe,
// lion_fp_probe and lion_unet_probe copy out: device pointers into the forward's arena, filled in by sa_fwd / fp_fwd /
// shared_mlp_fwd when Fwd::rec is set (never in a product call).
constexpr int MLP_REC_MAX = 4;
struct MlpRecord {
  int force = 0;                  // in: 0 = the path sa_fwd chooses, 1 = unfused kernels, 2 = fused (sa_fused.cu)
  bool fused = false;             // out: the path that ran
  int n = 0;                      // layers recorded
  const double* ssum[MLP_REC_MAX]; const double* ssq[MLP_REC_MAX]; int stat_stride[MLP_REC_MAX];
  const float* scale[MLP_REC_MAX]; const float* shift[MLP_REC_MAX];   // [B][C] folded AdaGN of each layer
  const float* pool_mm = nullptr; // last layer: [B][C/4][M][2][4] pre-activation minimum / maximum over the 32 neighbours
  // unpooled layers: the raw 1x1 output (PF of C/4 groups) and the activated output, at act_off of act_G groups
  const float4* raw[MLP_REC_MAX] = {}; const float4* act[MLP_REC_MAX] = {}; int act_G[MLP_REC_MAX] = {}, act_off[MLP_REC_MAX] = {};
  const float4* cat = nullptr;    // FP module: the MLP input [interpolated | skip] (PF)
};
// Caller buffers (device) that lion_unet_probe has unet_forward fill.  The U-Net releases arena marks between stages,
// so each result is copied out on the main stream where it is recorded, in the real pass only; a side-stream result
// (3-NN, time embedding) only after the main stream's wait for its event.  PFs are copied in their packed layout
// [B][G][R][4], the 3-NN in its [B][N][3] layout.  Any pointer may be null.
constexpr int UNET_REC_FP = 8;
struct UnetRecord {
  float *sinu = nullptr, *h = nullptr, *temb = nullptr, *aff = nullptr;   // [B][E] x 3, [B][style_total]
  struct Stage { float *cf, *nn_wgt, *skip, *cat, *out; int* nn_idx; } fp[UNET_REC_FP] = {};
  float *feat = nullptr, *cls_raw = nullptr, *cls_aff = nullptr, *hc = nullptr;   // head; cls_aff [2][B][128]
  double* cls_sums = nullptr;     // [2][B][128]
  int stage = 0;                  // the FP stage running
  const float *a_sinu = nullptr, *a_h = nullptr;                   // arena: the first two time-embedding stages
};
// Intermediate results of one PVConv (and its attention) that lion_pvconv_probe / lion_attention_probe copy out: device
// pointers into the forward's arena, filled in by pvconv_fwd / attn_fwd when Fwd::pv is set (never in a product call).
// In that mode pvconv_fwd also fills its raw1, act1 and raw2 grids with NaNs (0xff bytes) before their producers run,
// so that a read of a halo row nobody wrote shows up instead of depending on what the arena held.
struct PvRecord {
  const float4 *raw1 = nullptr, *act1 = nullptr, *raw2 = nullptr;   // VGs of cout channels (act1: halo included)
  bool act1_f16 = false;          // act1 holds rows of 8 halves (FP16 second convolution)
  const float4 *rawp = nullptr, *fused = nullptr;                    // PFs: point-branch 1x1 output, devox + point branch
  AffSrc a1{}, ap{}, a2{};        // AdaGN-1, point-branch AdaGN, AdaGN-2 with the SE gate: sums and folded scale / shift
  int conv2 = -1;                 // 0 = SIMT, 1 = tensor-core row tiles, 2 / 4 = interior-block groups of that many blocks
  const float4 *qkv = nullptr, *o = nullptr;                         // attention: PFs of 3 H 32 and H 32 channels
};
struct Fwd {
  Ctx* c; Model* m; int B;
  char* stat_pool = nullptr;     // all GroupNorm statistics of a forward: zeroed by ONE memset
  size_t stat_off = 0, stat_cap = 0;
  float* aff = nullptr;          // [B][style_total] all AdaGN (factor|bias) vectors of this forward
  std::deque<VoxPrep> vox;       // a deque: get_vox hands out pointers that later preps must not move
  MlpRecord* rec = nullptr;      // test entry points only
  PvRecord* pv = nullptr;        // test entry points only
  UnetRecord* ur = nullptr;      // test entry points only
  bool conv_f16 = false;         // LION_FWD_CONV_FP16: the PVConvs' second convolutions take FP16 operands (pvconv_fwd)
};
static bool record_layer(Fwd& f, const AffSrc& a) {
  MlpRecord* r = f.rec;
  if (!r || r->n >= MLP_REC_MAX) return false;
  r->ssum[r->n] = a.ssum; r->ssq[r->n] = a.ssq; r->stat_stride[r->n] = a.stat_stride;
  r->scale[r->n] = a.scale; r->shift[r->n] = a.shift;
  r->n++;
  return true;
}
// lion_unet_probe: copy `bytes` from the arena into a caller buffer now, on the main stream (real pass only)
static int rec_copy(Fwd& f, void* dst, const void* src, size_t bytes) {
  if (!dst || f.c->dry || !bytes) return 0;
  LION_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, f.c->stream));
  return 0;
}
static size_t pf_bytes(const Fwd& f, const PF& p) { return sizeof(float4) * f.B * p.G * p.R; }
// One point level of a forward: SA level i's input points, the centres its FPS samples from them (the points of
// level i + 1) with their ball-query neighbours, and the 3-NN of the points among the centres that the FP stage
// interpolating back onto them uses.  An event is set from the side stream's record of the result until the main
// stream has waited for it (wait_once).
struct Level {
  const float4* pts = nullptr; int n = 0;
  PF feat;                                        // features at pts (the FP stage's skip input)
  float4* centers = nullptr; int m = 0;
  int* nidx = nullptr;                            // [B][m][k]
  int* nn_idx = nullptr; float* nn_wgt = nullptr;  // [B][n][3]
  cudaEvent_t sa_done = nullptr, vox_done = nullptr, nn_done = nullptr;   // centres + nidx, voxel preps of pts, nn_*
};

static PF alloc_pf(Fwd& f, int G, int R) {
  PF t; t.G = G; t.R = R;
  t.p = f.c->alloc_n<float4>((size_t)f.B * G * R);
  return t;
}
// VG with guard rows on both sides (shifted conv reads may touch up to rp*rp+rp+1 rows outside)
static float4* alloc_vg(Fwd& f, int G, int r) {
  int rp = r + 2;
  size_t P = (size_t)rp * rp * rp, guard = (size_t)rp * rp + rp + 8;
  float4* base = f.c->alloc_n<float4>((size_t)f.B * G * P + 2 * guard);
  return base + guard;
}
// probe mode (Fwd::pv): every float of the VG's B * G * (r+2)^3 rows becomes a NaN
static int poison_vg(Fwd& f, float4* vg, int G, int r) {
  if (!f.pv) return 0;
  const size_t rp = r + 2;
  return memset_async(f.c, vg, 0xff, sizeof(float4) * f.B * G * rp * rp * rp);
}

static int style_affine_all(Fwd& f, const float* style) {
  Model* m = f.m;
  if (m->style_layers.empty()) return 0;
  f.aff = f.c->alloc_n<float>((size_t)f.B * m->style_total);
  LION_LAUNCH(f.c, k_style_linear, dim3((unsigned)m->style_layers.size(), f.B), 256, m->S * sizeof(float),
              m->d_style_layers, style, m->S, f.aff, m->style_total);
  return check_launch(f.c, "style_affine_all");
}

static ConvGeom geom_rows(int R) {
  ConvGeom g{};
  g.ntaps = 1; g.off[0] = 0; g.rp = 0; g.rows = R; g.p_begin = 0; g.p_end = R;
  g.occ = nullptr; g.occ_stride = 0;
  return g;
}
static ConvGeom geom_grid(int r) {
  ConvGeom g{};
  int rp = r + 2;
  g.ntaps = 27; g.rp = rp; g.rows = rp * rp * rp;
  for (int kx = 0; kx < 3; ++kx) for (int ky = 0; ky < 3; ++ky) for (int kz = 0; kz < 3; ++kz)
    g.off[(kx * 3 + ky) * 3 + kz] = (kx - 1) * rp * rp + (ky - 1) * rp + (kz - 1);
  g.p_begin = rp * rp; g.p_end = (rp - 1) * rp * rp;
  g.occ = nullptr; g.occ_stride = 0;
  return g;
}

// out rows in [p_begin,p_end) of every (b, group < Gout_store); statistics optional
// f16: the input is [Gin = C/8][rows][8] halves and the FP16 kernel runs (w.tc16 must exist)
static int run_conv(Fwd& f, const ConvW& w, const float4* in, int Gin, float4* out, int Gout_store,
                    double* ssum, double* ssq, const ConvGeom& geo, float* pool_mm = nullptr, bool f16 = false) {
  const int cpg = f16 ? 8 : 4;
  if (Gin * cpg != w.cin_pad) { set_error("conv: input has %d channels, weights expect %d", Gin * cpg, w.cin_pad); return LION_ERR_ARG; }
  if (f16) return conv_tc_run(f.c, w, in, Gin, out, Gout_store, ssum, ssq, geo, f.B, pool_mm, true);
  if (conv_tc_usable(w, geo))
    return conv_tc_run(f.c, w, in, Gin, out, Gout_store, ssum, ssq, geo, f.B, pool_mm);
  if (pool_mm) { set_error("conv: the pooled epilogue exists on the tensor-core path only"); return LION_ERR_STATE; }
  int span = geo.p_end - geo.p_begin;
  if (w.cout_pad == 4) {
    LION_LAUNCH(f.c, k_conv_simt<4>, dim3(cdiv(span, 128), 1, f.B), 128, geo.ntaps * 16 * sizeof(float),
                in, w.wt, w.bias, out, ssum, ssq, Gin, w.cin_pad, w.cout_pad, Gout_store, geo);
  } else {
    LION_LAUNCH(f.c, k_conv_simt<8>, dim3(cdiv(span, 128), w.cout_pad / 8, f.B), 128, geo.ntaps * 32 * sizeof(float),
                in, w.wt, w.bias, out, ssum, ssq, Gin, w.cin_pad, w.cout_pad, Gout_store, geo);
  }
  return check_launch(f.c, "conv");
}

// AdaGN (+SE) folded into y = scale*x + shift: k_affine_prep materialises the two [B][C] arrays per layer.
static PrepJob prep_job(Fwd& f, const AdaGNW& g, const double* ssum, const double* ssq, int stat_stride, double count,
                        const float* se1, const float* se2, AffSrc& a) {
  a = AffSrc{nullptr, nullptr, ssum, ssq, stat_stride, g.gamma, g.beta, f.aff + g.style_off, f.m->style_total, count};
  float* scale = f.c->alloc_n<float>((size_t)f.B * g.C);
  float* shift = f.c->alloc_n<float>((size_t)f.B * g.C);
  a.scale = scale; a.shift = shift;
  return PrepJob{ssum, ssq, stat_stride, g.gamma, g.beta, f.aff + g.style_off, f.m->style_total, se1, se2, scale, shift, g.C, count};
}
static int run_prep(Fwd& f, const PrepJob& j0, const PrepJob* j1) {
  int C = j0.C, njobs = 1;
  size_t smem = j0.se_w1 ? (j0.C + j0.C / 8) * sizeof(float) : 0;
  if (j1) {
    njobs = 2;
    if (j1->C > C) C = j1->C;
    size_t s1 = j1->se_w1 ? (j1->C + j1->C / 8) * sizeof(float) : 0;
    if (s1 > smem) smem = s1;
  }
  LION_LAUNCH(f.c, k_affine_prep, dim3(f.B, njobs), C, smem, j0, j1 ? *j1 : j0);
  return check_launch(f.c, "affine_prep");
}
static int run_affine(Fwd& f, const AdaGNW& g, const double* ssum, const double* ssq, int stat_stride, double count,
                      const float* se1, const float* se2, AffSrc& a) {
  PrepJob j = prep_job(f, g, ssum, ssq, stat_stride, count, se1, se2, a);
  return run_prep(f, j, nullptr);
}
static int stat_pool_begin(Fwd& f, size_t bytes) {
  f.stat_pool = (char*)f.c->alloc(bytes);
  f.stat_cap = bytes; f.stat_off = 0;
  return memset_async(f.c, f.stat_pool, 0, bytes);
}
static int alloc_stats(Fwd& f, int stride, double** ssum, double** ssq) {
  size_t bytes = sizeof(double) * 2 * f.B * stride;
  double* s;
  if (f.stat_pool && f.stat_off + bytes <= f.stat_cap) {        // pooled: already zero
    s = (double*)(f.stat_pool + f.stat_off);
    f.stat_off += bytes;
    *ssum = s; *ssq = s + (size_t)f.B * stride;
    return 0;
  }
  s = f.c->alloc_n<double>((size_t)2 * f.B * stride);
  *ssum = s; *ssq = s + (size_t)f.B * stride;
  return memset_async(f.c, s, 0, bytes);
}

// convolution + GroupNorm statistics (epilogue) + AdaGN(/SE) fold (k_affine_prep).
// Computing the fold in the LAST CTA of the convolution instead (arrival ticket, no extra launch) measured 1.3-2.0 ms
// per step SLOWER at B = 32 on the B200, before the port to H100 -- a single SM folding 2048-4096 (b, c) pairs with cold
// code on the critical path loses to a 32-CTA kernel whose launch latency the graph mostly hides -- so the separate
// launch stays.
static int conv_gn(Fwd& f, const ConvW& w, const float4* in, int Gin, float4* out, int Gout_store, const ConvGeom& geo,
                   const AdaGNW& g, double count, const float* se1, const float* se2, AffSrc& a, bool f16 = false) {
  double *ssum, *ssq;
  LION_TRY(alloc_stats(f, w.cout_pad, &ssum, &ssq));
  LION_TRY(run_conv(f, w, in, Gin, out, Gout_store, ssum, ssq, geo, nullptr, f16));
  return run_affine(f, g, ssum, ssq, w.cout_pad, count, se1, se2, a);
}
// same, but the fold is left to the caller (who merges it with another layer's: run_prep)
static int conv_gn_deferred(Fwd& f, const ConvW& w, const float4* in, int Gin, float4* out, int Gout_store, const ConvGeom& geo,
                            const AdaGNW& g, double count, AffSrc& a, PrepJob& job) {
  double *ssum, *ssq;
  LION_TRY(alloc_stats(f, w.cout_pad, &ssum, &ssq));
  LION_TRY(run_conv(f, w, in, Gin, out, Gout_store, ssum, ssq, geo));
  job = prep_job(f, g, ssum, ssq, w.cout_pad, count, nullptr, nullptr, a);
  return 0;
}

// SharedMLP on a PF.  pool: 1, or 32 = max over neighbour rows after the last activation.
// The activated result goes to dst (Gd groups, offset g_off, R/pool rows).
static int shared_mlp_fwd(Fwd& f, const SharedMLPBlk& m, PF in, int pool, float4* dst, int Gd, int g_off) {
  int n = (int)m.conv.size();
  PF cur = in;
  for (int i = 0; i < n; ++i) {
    const ConvW& w = m.conv[i];
    int Gout = w.cout / 4;
    bool last = (i == n - 1);
    AffSrc a;
    if (last && pool == 32 && cur.R % 128 == 0 && w.cout == w.cout_pad && conv_tc_usable(w, geom_rows(cur.R))) {
      // pooled last layer: the convolution's epilogue keeps, per centre and channel, the minimum and the maximum over the
      // 32 neighbours (enough to evaluate max_i swish(affine(x_i)) exactly, see conv_tc.cu: Params::pool_mm); the
      // [B, C, M, 32] tensor is never written
      int Ro = cur.R / 32;
      float* mm = f.c->alloc_n<float>((size_t)f.B * Gout * Ro * 8);
      double *ssum, *ssq;
      LION_TRY(alloc_stats(f, w.cout_pad, &ssum, &ssq));
      LION_TRY(run_conv(f, w, cur.p, cur.G, nullptr, Gout, ssum, ssq, geom_rows(cur.R), mm));
      LION_TRY(run_affine(f, m.gn[i], ssum, ssq, w.cout_pad, (double)cur.R, nullptr, nullptr, a));
      record_layer(f, a);
      if (f.rec) f.rec->pool_mm = mm;
      LION_LAUNCH(f.c, k_act_pool_minmax, dim3(cdiv(Ro, 256), Gout, f.B), 256, 0, (const float4*)mm, dst, a, Gout, w.cout, Ro, Gd, g_off);
      LION_TRY(check_launch(f.c, "shared_mlp pooled"));
      continue;
    }
    PF raw = alloc_pf(f, Gout, cur.R);
    LION_TRY(conv_gn(f, w, cur.p, cur.G, raw.p, Gout, geom_rows(cur.R), m.gn[i], (double)cur.R, nullptr, nullptr, a));
    const int l = record_layer(f, a) ? f.rec->n - 1 : -1;
    if (l >= 0) f.rec->raw[l] = raw.p;
    if (last && pool > 1) {
      if (pool != 32 || cur.R % 32) { set_error("shared_mlp: unsupported pooling %d", pool); return LION_ERR_ARG; }
      int Ro = cur.R / 32;
      LION_LAUNCH(f.c, k_act_rows_pool32, dim3(cdiv(Ro, 8 * 4), Gout, f.B), 256, 0, raw.p, dst, a, Gout, w.cout, Ro, Gd, g_off);
    } else {
      PF nxt;
      float4* o; int gd, go;
      if (last) { o = dst; gd = Gd; go = g_off; }
      else { nxt = alloc_pf(f, Gout, cur.R); o = nxt.p; gd = Gout; go = 0; }
      LION_LAUNCH(f.c, k_act_rows<1>, dim3(cdiv(cur.R, 256), Gout, f.B), 256, 0, raw.p, o, a, Gout, w.cout, cur.R, gd, go, last ? 0 : 1);
      if (l >= 0) { f.rec->act[l] = o; f.rec->act_G[l] = gd; f.rec->act_off[l] = go; }
      cur = nxt;
    }
    LION_TRY(check_launch(f.c, "shared_mlp act"));
  }
  return 0;
}

static int attn_fwd(Fwd& f, const AttnBlk& a, PF x, float4* dst, int Gd, int g_off) {
  int hid = a.heads * 32, N = x.R;
  PF qkv = alloc_pf(f, 3 * hid / 4, N);
  LION_TRY(run_conv(f, a.qkv, x.p, x.G, qkv.p, qkv.G, nullptr, nullptr, geom_rows(N)));
  const int S = cdiv(N, ATTN_CHUNK);
  if (S > 32) { set_error("attention: N=%d too large (max %d points)", N, 32 * ATTN_CHUNK); return LION_ERR_ARG; }
  float* part = f.c->alloc_n<float>((size_t)f.B * a.heads * S * ATTN_PART);
  LION_LAUNCH(f.c, k_attn_ctx, dim3(a.heads, f.B, S), 256, 0, qkv.p, part, a.heads, N);
  PF o = alloc_pf(f, hid / 4, N);
  LION_LAUNCH(f.c, k_attn_apply, dim3(cdiv(N, 128), a.heads, f.B), 128, 0, qkv.p, part, o.p, a.heads, N, S);
  LION_TRY(check_launch(f.c, "attention"));
  if (f.pv) { f.pv->qkv = qkv.p; f.pv->o = o.p; }
  if (Gd != a.C / 4 || g_off != 0) { set_error("attention: destination must be a plain PF"); return LION_ERR_ARG; }
  return run_conv(f, a.out, o.p, o.G, dst, a.C / 4, nullptr, nullptr, geom_rows(N));
}

// The first convolution of a PVConv reads a grid with at most N occupied voxels.  When that is a small fraction of r^3
// (<= 25 %) it is cheaper to multiply only the occupied voxels by all 27 taps (one GEMM, 27 * N rows of output instead of r^3 * 27
// taps of dense work) and let every output voxel gather its neighbours' rows (k_sparse_conv_gather): at r = 32, N = 2048
// that is 16x fewer FLOPs and the convolution becomes a ~0.7 GB streaming problem.
static bool sparse_conv1_wanted(int N, int r) {
  return (long long)N * 4 <= (long long)r * r * r;
}
// voxelisation prep of the points c4 at resolution r, launched on stream s (once per forward: later calls find it)
static int get_vox(Fwd& f, cudaStream_t s, const float4* c4, int N, int r, VoxPrep** out) {
  for (auto& v : f.vox) if (v.c4 == c4 && v.N == N && v.r == r) { *out = &v; return 0; }
  VoxPrep v{c4, N, r, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr};
  if (N > VOXP_MAXN || r > 32) { set_error("voxelisation: N=%d (max %d) or r=%d (max 32) unsupported", N, VOXP_MAXN, r); return LION_ERR_ARG; }
  v.nc = f.c->alloc_n<float4>((size_t)f.B * N);
  v.order = f.c->alloc_n<int>((size_t)f.B * N);
  v.ppos = f.c->alloc_n<int>((size_t)f.B * N);
  v.len = f.c->alloc_n<int>((size_t)f.B * N);
  int P = (r + 2) * (r + 2) * (r + 2);
  v.occ_stride = (P + 63) / 64 + 4;
  v.occ = f.c->alloc_n<unsigned char>((size_t)f.B * v.occ_stride);
  LION_TRY(memset_async(f.c, v.occ, 0, (size_t)f.B * v.occ_stride, s));
  if (sparse_conv1_wanted(N, r)) {
    v.cidx = f.c->alloc_n<int>((size_t)f.B * N);
    v.nocc = f.c->alloc_n<int>((size_t)f.B);
    v.vgrid = f.c->alloc_n<int>((size_t)f.B * P);
    LION_TRY(memset_async(f.c, v.vgrid, 0xff, (size_t)f.B * P * sizeof(int), s));     // -1 = empty voxel
  }
  LION_LAUNCH_ON(f.c, s, k_vox_prep, f.B, VOXP_THREADS, 0, c4, v.nc, v.order, v.ppos, v.len, v.occ, v.occ_stride, N, r, v.cidx, v.nocc,
                 v.vgrid);
  LION_TRY(check_launch(f.c, "vox_prep"));
  f.vox.push_back(v);
  *out = &f.vox.back();
  return 0;
}

// The first convolution of a PVConv, scatter included: the raw output (a VG of cout channels) and its GroupNorm sums.
// path: 0 = the product's choice (sparse when the grid is sparse enough and the wide packing serves it), 1 = the dense
// tensor-core convolution with occupancy skip, 2 = sparse.  A dense run leaves the scattered voxels in the context's zero
// grid (g_in): the caller restores it (k_act_grid's extra blocks).  after_scatter() runs between the scatter and the
// convolution (pvconv_fwd launches its point branch there).  A sparse run stores only the voxels its activity mask marks
// (the rest hold exactly the bias, which k_act_grid substitutes) unless whole_raw: then the raw output is stored whole.
// o.mask: the activity mask of a sparse run, [B][ceil(r^3 / 32)] words (null after a dense run).
struct Conv1Out { float4* raw = nullptr; double* ssum = nullptr; double* ssq = nullptr; float4* g_in = nullptr; bool sparse = false;
                  const unsigned* mask = nullptr; };
template <typename F>
static int pvconv_conv1(Fwd& f, const PVConvBlk& p, PF feat, const VoxPrep* vp, int path, bool whole_raw, Conv1Out& o,
                        F&& after_scatter) {
  const int N = feat.R, r = p.r, rp = r + 2, P = rp * rp * rp, Gin = p.cin / 4, Gout = p.cout / 4;
  ConvGeom geo1 = geom_grid(r);
  // (the tensor-core kernel still skips operand slabs whose 64-row occupancy flags are all clear)
  geo1.occ = vp->occ; geo1.occ_stride = vp->occ_stride;
  const bool sparse_ok = vp->cidx && ygemm_usable(p.c1y) && feat.G == p.c1y.cin_pad / 4;
  if (path == 2 && !sparse_ok) { set_error("PVConv: the sparse first convolution cannot serve this layer / grid"); return LION_ERR_ARG; }
  if (path == 1 && !conv_tc_usable(p.c1, geo1)) { set_error("PVConv: no tensor-core packing of the first convolution"); return LION_ERR_ARG; }
  const bool sparse1 = path == 0 ? sparse_ok : path == 2;
  o.sparse = sparse1;
  PF xc;
  if (sparse1) {
    // compact list of the occupied voxels' mean features (same values k_scatter would store into the grid)
    xc = alloc_pf(f, Gin, N);
    LION_LAUNCH(f.c, k_scatter_compact, dim3(cdiv(N, 128), Gin, f.B), 128, 0, feat.p, vp->order, vp->cidx, vp->len, vp->nocc, xc.p, Gin, N);
  } else {
    // point -> voxel scatter-mean into the context's persistent all-zero grid (no per-call memset)
    size_t zbytes = sizeof(float4) * ((size_t)f.B * Gin * P + 2 * ((size_t)rp * rp + rp + 8));
    if (zbytes > f.c->zgrid_need) f.c->zgrid_need = zbytes;
    o.g_in = f.c->dry ? (float4*)(uintptr_t)0x1000 : (float4*)f.c->zgrid + ((size_t)rp * rp + rp + 8);
    LION_LAUNCH(f.c, k_scatter, dim3(cdiv(N, 128), Gin, f.B), 128, 0, feat.p, vp->order, vp->ppos, vp->len, o.g_in, Gin, N, P);
  }
  stamp(f.c, f.c->stream, " scatter");
  LION_TRY(after_scatter());
  float4* raw1 = alloc_vg(f, Gout, r);
  o.raw = raw1;
  LION_TRY(poison_vg(f, raw1, Gout, r));
  if (sparse1) {
    const int ld = 27 * p.c1.cout_pad;
    float* y = f.c->alloc_n<float>((size_t)f.B * N * ld);
    LION_TRY(ygemm_run(f.c, p.c1y, xc.p, y, ld, vp->nocc, f.B, N));
    double *s1, *q1;
    LION_TRY(alloc_stats(f, p.c1.cout_pad, &s1, &q1));
    const int nwarp = 4;
    const size_t smem = (size_t)nwarp * (32 * (p.c1.cout_pad + 2) * sizeof(float) + SPG_LIST * sizeof(unsigned));
    static DevOnce attr_once;
    if (attr_once.need()) {
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_sparse_conv_gather<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_sparse_conv_gather<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
      // level 0 runs next to the side stream: same (maximum) shared-memory carve-out as its kernels, or these blocks
      // cannot become resident on the SMs FPS occupies (see unet_forward)
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_sparse_conv_gather<32>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_sparse_conv_gather<64>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_act_grid<false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_act_grid<true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_scatter_compact, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
    const dim3 grid(cdiv(r * r * r, 32 * nwarp), f.B);
    unsigned* mask = f.c->alloc_n<unsigned>((size_t)f.B * cdiv(r * r * r, 32));
    const bool whole = whole_raw || f.c->sparse_conv1_dense;
    if (p.c1.cout_pad == 32)
      LION_LAUNCH(f.c, k_sparse_conv_gather<32>, grid, 32 * nwarp, smem, y, ld, vp->vgrid, p.c1.bias, raw1, s1, q1, p.c1.cout_pad, r, N,
                  mask, whole);
    else
      LION_LAUNCH(f.c, k_sparse_conv_gather<64>, grid, 32 * nwarp, smem, y, ld, vp->vgrid, p.c1.bias, raw1, s1, q1, p.c1.cout_pad, r, N,
                  mask, whole);
    LION_TRY(check_launch(f.c, "sparse conv1"));
    o.ssum = s1; o.ssq = q1;
    o.mask = mask;
  } else {
    LION_TRY(alloc_stats(f, p.c1.cout_pad, &o.ssum, &o.ssq));
    LION_TRY(run_conv(f, p.c1, o.g_in, Gin, raw1, Gout, o.ssum, o.ssq, geo1));
  }
  return 0;
}

// The second convolution of a PVConv whose first one ran sparse reads, at every interior voxel without an occupied
// neighbour (mask1 clear), the one value per (shape, channel) that k_act_grid writes there.  An output voxel none of
// whose 27 neighbours is active is then a function of its border class alone (low, interior or high in each of x, y and
// z): k_conv2_flags marks the row tiles' 64-row blocks made only of such voxels, and the same kernel instantiation
// convolves a 3x3x3 grid of that value (k_act_grid with an all-clear mask, so the very same bits) into the 27 class
// values per channel.  The tensor cores give an output element the same bits whatever its row, so the convolution
// can skip those blocks' copies and MMAs and take their outputs and GroupNorm sums from the class values
// (conv_tc.cu: Params::cls_flag) without changing a bit.  Flagged rows are stored in probe mode only: the
// devoxelisation reads trilinear corners within one voxel of a point, which are active.
static int conv2_classes(Fwd& f, const PVConvBlk& p, const VoxPrep* vp, const unsigned* mask1, const float4* raw1,
                         const AffSrc& a1, bool h2, ConvGeom& geo) {
  const int r = p.r, rp = r + 2, Gout = p.cout / 4, Gc = p.c2.cout_pad / 4, Gact = h2 ? Gout / 2 : Gout;
  const int nblk = 2 * cdiv(r * rp * rp, 128);        // two per row tile
  if (nblk > vp->occ_stride) { set_error("conv2 classes: %d blocks exceed the flag stride %d", nblk, vp->occ_stride); return LION_ERR_STATE; }
  unsigned char* flags = f.c->alloc_n<unsigned char>((size_t)f.B * vp->occ_stride);
  unsigned* zmask = f.c->alloc_n<unsigned>((size_t)f.B);
  LION_TRY(memset_async(f.c, f.c->d_cls_count, 0, sizeof(unsigned long long)));
  LION_LAUNCH(f.c, k_conv2_flags, dim3(cdiv(nblk, 8), f.B), 256, 0, mask1, r, nblk, flags, vp->occ_stride, zmask, f.c->d_cls_count);
  f.c->cls_blocks = (long long)f.B * nblk;
  // the class grid (r = 3, 125 rows per channel group); its row tile reads from 31 rows before to 59 past them, whose
  // outputs are not kept
  const int CP = 125, guard = 64;
  float4* cg = f.c->alloc_n<float4>((size_t)f.B * Gact * CP + 2 * guard) + guard;
  if (h2)
    LION_LAUNCH(f.c, k_act_grid<true>, dim3(1, Gact, f.B), 256, 0, raw1, cg, a1, Gout, p.cout, 5, CP, 1, nullptr, nullptr, 0, 0,
                zmask, p.c1.bias);
  else
    LION_LAUNCH(f.c, k_act_grid<false>, dim3(1, Gact, f.B), 256, 0, raw1, cg, a1, Gout, p.cout, 5, CP, 1, nullptr, nullptr, 0, 0,
                zmask, p.c1.bias);
  LION_TRY(check_launch(f.c, "conv2 classes"));
  float4* cls = f.c->alloc_n<float4>((size_t)f.B * Gc * CP);
  LION_TRY(run_conv(f, p.c2, cg, Gact, cls, Gc, nullptr, nullptr, geom_grid(3), nullptr, h2));
  geo.cls_flag = flags; geo.cls_stride = vp->occ_stride; geo.cls = cls; geo.cls_store = f.pv != nullptr;
  return 0;
}

// PVConv: features PF [cin] + coords -> dst PF (cout) at (Gd, g_off)
static int pvconv_fwd(Fwd& f, const PVConvBlk& p, PF feat, const float4* c4, float4* dst, int Gd, int g_off) {
  int N = feat.R, r = p.r, rp = r + 2, P = rp * rp * rp, Gin = p.cin / 4, Gout = p.cout / 4;
  if (feat.G != Gin) { set_error("PVConv: got %d input channels, expected %d", feat.G * 4, p.cin); return LION_ERR_ARG; }
  VoxPrep* vp;
  LION_TRY(get_vox(f, f.c->stream, c4, N, r, &vp));
  size_t mk = f.c->mark();
  ConvGeom geo = geom_grid(r);
  const ConvW& pw = p.point.conv[0];
  PF rawp;
  AffSrc ap;
  PrepJob jp, j1;
  // scatter -> point branch -> conv1 -> (stats) -> AdaGN + Swish.  The point branch is conv1x1 -> stats (its fold shares
  // a launch with conv1's below; the activation is applied inside the devox kernel).
  Conv1Out c1;
  LION_TRY(pvconv_conv1(f, p, feat, vp, 0, f.pv != nullptr, c1, [&]() -> int {
    rawp = alloc_pf(f, Gout, N);
    return conv_gn_deferred(f, pw, feat.p, feat.G, rawp.p, Gout, geom_rows(N), p.point.gn[0], (double)N, ap, jp);
  }));
  const bool sparse1 = c1.sparse;
  float4 *raw1 = c1.raw, *g_in = c1.g_in;
  const unsigned* mask1 = f.c->sparse_conv1_dense ? nullptr : c1.mask;     // (null: k_act_grid reads every position)
  AffSrc a1;
  const double V = (double)r * r * r;
  j1 = prep_job(f, p.g1, c1.ssum, c1.ssq, p.c1.cout_pad, V, nullptr, nullptr, a1);
  LION_TRY(run_prep(f, j1, &jp));
  stamp(f.c, f.c->stream, " conv1");
  // AdaGN-1 + Swish as a stand-alone pass over the grid (HBM-bound).  Folding it into conv2's operand staging
  // ("transform on load") was parity-green but made the convolutions 3.5x slower (measured on the B200, before the
  // port to H100).  Its extra blocks re-zero the scatter grid (was: k_unscatter).  FP16 mode (where the FP16 kernel
  // serves conv2): the grid is [C/8][P][8] halves, half the bytes, and conv2 takes FP16 operands.
  const bool h2 = f.conv_f16 && p.c2.tc16.w;
  const int Gact = h2 ? Gout / 2 : Gout;
  float4* act1 = alloc_vg(f, Gact, r);
  LION_TRY(poison_vg(f, act1, Gact, r));
  {
    const int nb_act = cdiv(P, 256 * ACT_U);
    const dim3 grid(nb_act + (sparse1 ? 0 : cdiv(N, 256)), Gact, f.B);
    if (h2)
      LION_LAUNCH(f.c, k_act_grid<true>, grid, 256, 0, raw1, act1, a1, Gout, p.cout, rp, P, nb_act, vp->ppos, g_in, Gin, N, mask1,
                  p.c1.bias);
    else
      LION_LAUNCH(f.c, k_act_grid<false>, grid, 256, 0, raw1, act1, a1, Gout, p.cout, rp, P, nb_act, vp->ppos, g_in, Gin, N, mask1,
                  p.c1.bias);
  }
  stamp(f.c, f.c->stream, " act1");
  // conv2 -> (stats) -> AdaGN + SE folded into one affine
  float4* raw2 = alloc_vg(f, Gout, r);
  LION_TRY(poison_vg(f, raw2, Gout, r));
  ConvGeom geo2 = geo;
  // (r >= 3: at r <= 2 a voxel lies on both the low and the high border and has no single class)
  if (mask1 && r >= 3 && f.c->conv2_class_mode != 1 && conv_tc_row_tiles_3x3(p.c2)) {
    if (f.c->conv2_class_mode == 2 && !f.pv)
      LION_TRY(memset_async(f.c, raw2, 0xff, sizeof(float4) * f.B * Gout * (size_t)P));
    LION_TRY(conv2_classes(f, p, vp, mask1, raw1, a1, h2, geo2));
  }
  AffSrc a2;
  LION_TRY(conv_gn(f, p.c2, act1, Gact, raw2, Gout, geo2, p.g2, V, p.se1, p.se2, a2, h2));
  stamp(f.c, f.c->stream, " conv2");
  if (f.pv) {
    PvRecord& R = *f.pv;
    R.raw1 = raw1; R.act1 = act1; R.raw2 = raw2; R.rawp = rawp.p; R.act1_f16 = h2;
    R.a1 = a1; R.ap = ap; R.a2 = a2;
    R.conv2 = !conv_tc_usable(p.c2, geo) ? 0 : f.c->conv_group_blocks ? f.c->conv_group_blocks : 1;
  }
  // voxel -> point gather (+ point branch)
  if (p.has_attn) {
    PF fused = alloc_pf(f, Gout, N);
    LION_LAUNCH(f.c, k_devox_fuse, dim3(cdiv(N, 128), Gout, f.B), 128, 0, raw2, vp->nc, a2.scale, a2.shift, rawp.p, ap,
                fused.p, Gout, p.cout, N, r, P, Gout, 0);
    LION_TRY(check_launch(f.c, "pvconv"));
    if (f.pv) f.pv->fused = fused.p;
    if (Gd != Gout || g_off != 0) {
      PF t = alloc_pf(f, Gout, N);
      LION_TRY(attn_fwd(f, p.attn, fused, t.p, Gout, 0));
      LION_LAUNCH(f.c, k_copy_groups, dim3(cdiv(N, 256), Gout, f.B), 256, 0, t.p, dst, Gout, Gd, g_off, N);
    } else {
      LION_TRY(attn_fwd(f, p.attn, fused, dst, Gd, g_off));
    }
  } else {
    LION_LAUNCH(f.c, k_devox_fuse, dim3(cdiv(N, 128), Gout, f.B), 128, 0, raw2, vp->nc, a2.scale, a2.shift, rawp.p, ap,
                dst, Gout, p.cout, N, r, P, Gd, g_off);
    if (f.pv) f.pv->fused = dst;    // (the probe's destination is a plain PF: Gd == Gout, g_off == 0)
  }
  LION_TRY(check_launch(f.c, "pvconv"));
  f.c->release(mk);   // grids are dead once the output PF is written (stream order keeps this safe)
  return 0;
}

// furthest-point sampling of M centres (and their indices) out of N packed points per shape, on stream s
template <int A, int C, bool FULL>
static int fps_c4_on(Ctx* c, cudaStream_t s, int B, const float4* c4, int* fidx, float4* centers, int N, int M, int VT) {
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_fps_c4<A, C, FULL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fps_smem_bytes(FPS_MAX_N)));
    // FPS runs on the side stream next to the convolutions: same (maximum) carve-out as theirs (see unet_forward)
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_fps_c4<A, C, FULL>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
  }
  LION_LAUNCH_ON(c, s, (k_fps_c4<A, C, FULL>), B, FPS_THREADS, fps_smem_bytes(N), c4, fidx, centers, N, M, VT);
  return 0;
}
static int fps_c4(Ctx* c, cudaStream_t s, int B, const float4* c4, int* fidx, float4* centers, int N, int M) {
  const int VT = fps_virtual_threads(N);
  int rc = 0;
#define LION_FPS_CALL(A_, C_, F_) rc = fps_c4_on<A_, C_, F_>(c, s, B, c4, fidx, centers, N, M, VT)
  LION_FPS_DISPATCH(N, VT, LION_FPS_CALL);
#undef LION_FPS_CALL
  return rc;
}

// the side stream records `e` once its result is complete and leaves it in `slot`; the main stream waits for it
// where it first needs the result, and only there
static int record_on_aux(Ctx* c, cudaEvent_t e, cudaEvent_t& slot) {
  if (!c->dry) { LION_CHECK_CUDA(cudaEventRecord(e, c->aux)); slot = e; }
  return 0;
}
static int wait_once(Ctx* c, cudaEvent_t& slot) {
  if (slot) LION_CHECK_CUDA(cudaStreamWaitEvent(c->stream, slot, 0));
  slot = nullptr;
  return 0;
}

// SA geometry of level i, on stream st: FPS of s.m centres out of lv.pts into lv.centers (allocated by the caller),
// then the ball query of the k neighbours of each centre
static int sa_geometry(Fwd& f, cudaStream_t st, const SABlk& s, Level& lv, int i) {
  const int N = lv.n, M = s.m;
  if (N > FPS_MAX_N) { set_error("SA: N=%d too large for FPS", N); return LION_ERR_ARG; }
  if (M > N) { set_error("SA: more centres (%d) than points (%d)", M, N); return LION_ERR_ARG; }
  lv.m = M;
  int* fidx = f.c->alloc_n<int>((size_t)f.B * M);
  LION_TRY(fps_c4(f.c, st, f.B, lv.pts, fidx, lv.centers, N, M));
  stamp(f.c, st, "fps", i);
  lv.nidx = f.c->alloc_n<int>((size_t)f.B * M * s.k);
  LION_LAUNCH_ON(f.c, st, k_ball_query_c4, dim3(cdiv(M * 32, 256), f.B), 256, 0, lv.centers, lv.pts, lv.nidx, N, M,
                 s.radius * s.radius, s.k);
  stamp(f.c, st, "ballq", i);
  return 0;
}
// FP geometry of level i, on stream st: the 3 nearest centres of every point and their interpolation weights
static int fp_geometry(Fwd& f, cudaStream_t st, Level& lv, int i) {
  lv.nn_idx = f.c->alloc_n<int>((size_t)f.B * lv.n * 3);
  lv.nn_wgt = f.c->alloc_n<float>((size_t)f.B * lv.n * 3);
  LION_LAUNCH_ON(f.c, st, k_three_nn_c4, dim3(cdiv(lv.n, 128), f.B), 128, 1024 * sizeof(float4), lv.pts, lv.centers, lv.nn_idx,
                 lv.nn_wgt, lv.n, lv.m);
  stamp(f.c, st, "3nn", i);
  return 0;
}

// SA module: features PF at lv.pts -> dst PF (Gd groups at g_off) at lv.centers
static int sa_fwd(Fwd& f, const SABlk& s, PF feat, Level& lv, float4* dst, int Gd, int g_off) {
  int N = feat.R, M = s.m, U = s.k, Gf = s.cfeat / 4;
  if (feat.G != Gf) { set_error("SA: got %d feature channels, expected %d", feat.G * 4, s.cfeat); return LION_ERR_ARG; }
  size_t mk = f.c->mark();
  LION_TRY(wait_once(f.c, lv.sa_done));
  if (sa_fused_usable(s) && !(f.rec && f.rec->force == 1)) {
    // gather -> conv -> AdaGN/Swish -> conv -> max-pool in two fused passes (sa_fused.cu): no [B, C, M, 32] round trips
    const ConvW &c1 = s.mlp.conv[0], &c2 = s.mlp.conv[1];
    double *s1, *q1, *s2, *q2;
    AffSrc a1, a2;
    LION_TRY(alloc_stats(f, c1.cout_pad, &s1, &q1));
    LION_TRY(sa_fused_run(f.c, s, feat.p, lv.pts, lv.centers, lv.nidx, nullptr, nullptr, s1, q1, c1.cout_pad, nullptr, f.B, N));
    LION_TRY(run_affine(f, s.mlp.gn[0], s1, q1, c1.cout_pad, (double)M * U, nullptr, nullptr, a1));
    LION_TRY(alloc_stats(f, c2.cout_pad, &s2, &q2));
    float* mm = f.c->alloc_n<float>((size_t)f.B * (c2.cout / 4) * M * 8);
    LION_TRY(sa_fused_run(f.c, s, feat.p, lv.pts, lv.centers, lv.nidx, a1.scale, a1.shift, s2, q2, c2.cout_pad, mm, f.B, N));
    LION_TRY(run_affine(f, s.mlp.gn[1], s2, q2, c2.cout_pad, (double)M * U, nullptr, nullptr, a2));
    if (f.rec) { record_layer(f, a1); record_layer(f, a2); f.rec->pool_mm = mm; f.rec->fused = true; }
    LION_LAUNCH(f.c, k_act_pool_minmax, dim3(cdiv(M, 256), c2.cout / 4, f.B), 256, 0, (const float4*)mm, dst, a2, c2.cout / 4, c2.cout, M,
                Gd, g_off);
    LION_TRY(check_launch(f.c, "sa fused"));
    f.c->release(mk);
    return 0;
  }
  PF grp = alloc_pf(f, Gf + 1, M * U);
  LION_LAUNCH(f.c, k_group_gather, dim3(cdiv(M * U, 256), Gf + 1, f.B), 256, 0, feat.p, lv.pts, lv.centers, lv.nidx, grp.p, Gf, N, M, U);
  LION_TRY(check_launch(f.c, "sa grouping"));
  LION_TRY(shared_mlp_fwd(f, s.mlp, grp, 32, dst, Gd, g_off));
  f.c->release(mk);
  return 0;
}

// FP module: interpolate the features at lv.centers (cfeat) to lv.pts, concat the skip features lv.feat, SharedMLP
static int fp_fwd(Fwd& f, const FPBlk& b, Level& lv, PF cfeat, float4* dst, int Gd, int g_off) {
  const int N = lv.n, M = lv.m, Gc = b.cc / 4, Gs = roundup(b.cp, 4) / 4;
  const PF& skip = lv.feat;
  if (cfeat.G != Gc || cfeat.R != M) { set_error("FP: centre features mismatch"); return LION_ERR_ARG; }
  if (Gs && (skip.G != Gs || skip.R != N)) { set_error("FP: skip features mismatch (%d groups, expected %d)", skip.G, Gs); return LION_ERR_ARG; }
  size_t mk = f.c->mark();
  LION_TRY(wait_once(f.c, lv.nn_done));
  PF cat = alloc_pf(f, Gc + Gs, N);
  // probe mode: every float of cat a NaN first, so that a row or channel nobody writes shows up
  if (f.rec || f.ur) LION_TRY(memset_async(f.c, cat.p, 0xff, pf_bytes(f, cat)));
  LION_LAUNCH(f.c, k_interp_rows, dim3(cdiv(N, 128), Gc, f.B), 128, 0, cfeat.p, lv.nn_idx, lv.nn_wgt, cat.p, Gc, M, N, Gc + Gs, 0);
  if (Gs) LION_LAUNCH(f.c, k_copy_groups, dim3(cdiv(N, 256), Gs, f.B), 256, 0, skip.p, cat.p, Gs, Gc + Gs, Gc, N);
  LION_TRY(check_launch(f.c, "fp interpolate"));
  if (f.rec) f.rec->cat = cat.p;
  if (f.ur) {
    UnetRecord::Stage& s = f.ur->fp[f.ur->stage];
    LION_TRY(rec_copy(f, s.nn_idx, lv.nn_idx, sizeof(int) * f.B * N * 3));
    LION_TRY(rec_copy(f, s.nn_wgt, lv.nn_wgt, sizeof(float) * f.B * N * 3));
    if (Gs) LION_TRY(rec_copy(f, s.skip, skip.p, pf_bytes(f, skip)));
    LION_TRY(rec_copy(f, s.cat, cat.p, pf_bytes(f, cat)));
  }
  LION_TRY(shared_mlp_fwd(f, b.mlp, cat, 1, dst, Gd, g_off));
  f.c->release(mk);
  return 0;
}

// SA level i: its PVConvs on lv.pts, then its SA module onto lv.centers; feat is the level's input and becomes its
// output.  Unless the caller has already planned the level's geometry (unet_forward, on the side stream), FPS and ball
// query run here on the main stream, just before the SA module.
static int sa_level_fwd(Fwd& f, const std::vector<Block>& blocks, Level& lv, PF& feat, int i) {
  for (auto& blk : blocks) {
    if (blk.kind == LION_KIND_PVCONV) {
      PF o = alloc_pf(f, blk.pv.cout / 4, lv.n);
      LION_TRY(pvconv_fwd(f, blk.pv, feat, lv.pts, o.p, o.G, 0));
      feat = o;
      stamp(f.c, f.c->stream, "sa.pvconv", i);
      continue;
    }
    PF o = alloc_pf(f, blk.sa.mlp.cout() / 4, blk.sa.m);
    const bool planned = lv.nidx != nullptr;
    if (!planned) lv.centers = f.c->alloc_n<float4>((size_t)f.B * blk.sa.m);
    const size_t mk = f.c->mark();
    if (!planned) LION_TRY(sa_geometry(f, f.c->stream, blk.sa, lv, i));
    LION_TRY(sa_fwd(f, blk.sa, feat, lv, o.p, o.G, 0));
    f.c->release(mk);
    feat = o;
    stamp(f.c, f.c->stream, "sa.module", i);
  }
  return 0;
}

// =====================================================================================
// U-Net
// =====================================================================================
static float bits_to_float(int v) { float f; memcpy(&f, &v, 4); return f; }

// desc: [num_classes, embed_dim, extra, input_dim, use_att, clip, clip_dim, S,
//        n_sa, {has_conv, oc, nblk, res, m, radius_bits, k, n_mlp, mlp...}*,
//        n_fp, {n_mlp, mlp..., has_conv, oc, nblk, res}*]
// The level/block structure restates create_pointnet2_sa_components / create_pointnet2_fp_modules
// (models/pvcnn2_ada.py:448-567) including their quirks (SURVEY.md Appendix A).
// the set-abstraction half of a PVCNN2 network: restates create_pointnet2_sa_components (models/pvcnn2_ada.py:448-517 and
// the non-Ada twin models/pvcnn2.py:440-509) including their quirk that levels > 0 keep only their first PVConv.
// Reads n_sa records {has_conv, oc, nblk, res, m, radius_bits, k, n_mlp, mlp...} from d at q.
static int build_sa_levels(Model* m, Cursor& cur, const std::vector<int>& d, size_t& q, int n_sa, int E, bool use_att, bool plain,
                           std::vector<std::vector<Block>>& levels, std::vector<int>& sa_in, int& in_ch) {
  auto rd = [&](int& v) { if (q >= d.size()) return false; v = d[q++]; return true; };
  for (int c = 0; c < n_sa; ++c) {
    int has_conv, oc, nblk, res, mc, rbits, kk, nm;
    if (!(rd(has_conv) && rd(oc) && rd(nblk) && rd(res) && rd(mc) && rd(rbits) && rd(kk) && rd(nm))) { set_error("descriptor truncated (sa)"); return LION_ERR_ARG; }
    std::vector<int> mlp(nm);
    for (int i = 0; i < nm; ++i) if (!rd(mlp[i])) { set_error("descriptor truncated (sa mlp)"); return LION_ERR_ARG; }
    std::vector<Block> blocks;
    sa_in.push_back(in_ch);
    int k = 0;
    if (has_conv) {
      for (int p = 0; p < nblk; ++p) {
        bool att = ((c + 1) % 2 == 0) && use_att && p == 0;
        if (c == 0 || k == 0) {
          blocks.emplace_back();
          blocks.back().kind = LION_KIND_PVCONV;
          LION_TRY(make_pvconv(m, blocks.back().pv, cur, (c == 0 || k > 0) ? in_ch : in_ch + E, oc, res, att, plain));
        }
        in_ch = oc;
        k++;
      }
    }
    int cfeat = in_ch + (k == 0 ? E : 0);
    blocks.emplace_back();
    blocks.back().kind = LION_KIND_SA;
    float radius; memcpy(&radius, &rbits, 4);
    LION_TRY(make_sa(m, blocks.back().sa, cur, cfeat, mc, radius, kk, mlp, plain));
    in_ch = mlp.back();
    levels.push_back(std::move(blocks));
  }
  return 0;
}

static int build_unet(Model* m, Cursor& cur) {
  const std::vector<int>& d = m->desc;
  size_t q = 0;
  auto rd = [&](int& v) { if (q >= d.size()) return false; v = d[q++]; return true; };
  m->unet.reset(new UnetBlk());
  UnetBlk& u = *m->unet;
  int n_sa = 0;
  if (!(rd(u.num_classes) && rd(u.embed_dim) && rd(u.extra) && rd(u.input_dim) && rd(u.use_att) && rd(u.clip) &&
        rd(u.clip_dim) && rd(u.S) && rd(n_sa))) { set_error("unet descriptor too short"); return LION_ERR_ARG; }
  if (n_sa < 1) { set_error("unet: at least one SA level"); return LION_ERR_ARG; }
  m->S = u.S;
  int E = u.embed_dim;
  if (u.input_dim != 3 || u.extra < 0 || u.extra > 1) { set_error("unet: points must be xyz + at most one extra feature channel"); return LION_ERR_ARG; }
  if (E % 4) { set_error("unet: embed_dim must be a multiple of 4"); return LION_ERR_ARG; }
  if (E > 0) {
    u.e0w = cur.next(); u.e0b = cur.next(); u.e2w = cur.next(); u.e2b = cur.next();
    int half = E / 2;
    std::vector<float> fr(half);
    for (int i = 0; i < half; ++i) fr[i] = (float)std::exp((double)i * -(std::log(10000.0) / (half - 1)));
    LION_TRY(m->dmalloc(&u.d_freqs, (size_t)half));
    LION_CHECK_CUDA(cudaMemcpy(u.d_freqs, fr.data(), half * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (u.clip) { u.cfw = cur.next(); u.cfb = cur.next(); u.scw = cur.next(); u.scb = cur.next(); }
  int in_ch = u.extra + u.input_dim;
  std::vector<int> sa_in;
  LION_TRY(build_sa_levels(m, cur, d, q, n_sa, E, u.use_att != 0, false, u.sa, sa_in, in_ch));
  int ch_sa = in_ch;
  sa_in[0] = u.extra + u.input_dim - 3;
  if (u.use_att) LION_TRY(make_attn(m, u.gatt, cur, ch_sa, 8));
  int n_fp = 0;
  if (!rd(n_fp)) { set_error("unet descriptor truncated (fp)"); return LION_ERR_ARG; }
  if (n_fp > n_sa) { set_error("unet: %d FP stages for %d SA levels", n_fp, n_sa); return LION_ERR_ARG; }
  for (int i = 0; i < n_fp; ++i) {
    int nm;
    if (!rd(nm)) { set_error("unet descriptor truncated (fp)"); return LION_ERR_ARG; }
    std::vector<int> mlp(nm);
    for (int j = 0; j < nm; ++j) if (!rd(mlp[j])) { set_error("unet descriptor truncated (fp mlp)"); return LION_ERR_ARG; }
    int has_conv, oc, nblk, res;
    if (!(rd(has_conv) && rd(oc) && rd(nblk) && rd(res))) { set_error("unet descriptor truncated (fp conv)"); return LION_ERR_ARG; }
    std::vector<Block> blocks;
    blocks.emplace_back();
    blocks.back().kind = LION_KIND_FP;
    LION_TRY(make_fp(m, blocks.back().fp, cur, in_ch + E, sa_in[n_sa - 1 - i], mlp));
    in_ch = mlp.back();
    if (has_conv) {
      for (int p = 0; p < nblk; ++p) {
        blocks.emplace_back();
        blocks.back().kind = LION_KIND_PVCONV;
        LION_TRY(make_pvconv(m, blocks.back().pv, cur, in_ch, oc, res, false));
        in_ch = oc;
      }
    }
    u.fp.push_back(std::move(blocks));
  }
  int scale_bits;
  if (!rd(scale_bits)) { set_error("unet descriptor truncated (time-embedding scale)"); return LION_ERR_ARG; }
  memcpy(&u.time_scale, &scale_bits, sizeof(float));
  // per point level: the voxel preps of the PVConvs on its points (SA level l's, then FP stage n_sa - 1 - l's) and the
  // events of what the side stream computes for it
  u.levels.resize(n_sa);
  for (int l = 0; l < n_sa; ++l) {
    UnetLevel& lv = u.levels[l];
    auto add_r = [&](const std::vector<Block>& blocks) {
      for (auto& b : blocks)
        if (b.kind == LION_KIND_PVCONV && std::find(lv.vox_r.begin(), lv.vox_r.end(), b.pv.r) == lv.vox_r.end()) lv.vox_r.push_back(b.pv.r);
    };
    add_r(u.sa[l]);
    if (n_sa - 1 - l < n_fp) add_r(u.fp[n_sa - 1 - l]);
    for (cudaEvent_t* e : {&lv.sa_done, &lv.vox_done, &lv.nn_done}) LION_TRY(m->make_event(e));
  }
  for (cudaEvent_t* e : {&u.aux_start, &u.temb_done}) LION_TRY(m->make_event(e));
  // classifier: SharedMLP(ch_fp -> 128), Dropout, Conv1d(128 -> num_classes) (latent_points_ada.py:94-99)
  LION_TRY(make_shared_mlp(m, u.cls0, cur, in_ch, ident_map(in_ch), {128}));
  const float* cw = cur.next(); const float* cb = cur.next();
  if (cur.bad) { set_error("unet: parameter list too short (%d given)", cur.n); return LION_ERR_ARG; }
  LION_TRY(make_conv(m, u.cls2, cw, cb, 1, 128, u.num_classes, ident_map(128)));
  if (cur.i != cur.n) { set_error("unet: %d parameters given, %d consumed", cur.n, cur.i); return LION_ERR_ARG; }
  return 0;
}

__global__ void k_extract_extra(const float4* __restrict__ x, float4* __restrict__ o, int total) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) o[i] = make_float4(x[i].w, 0.f, 0.f, 0.f);
}

// descriptor [input_dim, zdim, use_att, n_sa, levels...]; parameters: the SA levels in state_dict order, then mlp.weight/bias
static int build_style_enc(Model* m, Cursor& cur) {
  const std::vector<int>& d = m->desc;
  if (d.size() < 4) { set_error("style encoder descriptor: [input_dim, zdim, use_att, n_sa, levels...]"); return LION_ERR_ARG; }
  m->senc.reset(new StyleEncBlk());
  StyleEncBlk& e = *m->senc;
  e.input_dim = d[0]; e.zdim = d[1];
  if (e.input_dim != 3) { set_error("style encoder: input_dim must be 3"); return LION_ERR_ARG; }
  size_t q = 4;
  int in_ch = e.input_dim;
  std::vector<int> sa_in;
  LION_TRY(build_sa_levels(m, cur, d, q, d[3], 0, d[2] != 0, true, e.sa, sa_in, in_ch));
  e.cfeat = in_ch;
  e.mlp_w = cur.next(); e.mlp_b = cur.next();
  if (cur.bad || cur.i != cur.n) { set_error("style encoder: %d parameters given, %d consumed", cur.n, cur.i); return LION_ERR_ARG; }
  if (e.cfeat % 4) { set_error("style encoder: feature width must be a multiple of 4"); return LION_ERR_ARG; }
  m->S = 4;   // no style input: every normalisation is a plain GroupNorm
  return 0;
}

static int style_enc_forward(Fwd& f, const float* x, float* out, int N) {
  StyleEncBlk& e = *f.m->senc;
  Ctx* c = f.c;
  int B = f.B;
  float4* c0 = c->alloc_n<float4>((size_t)B * N);
  LION_LAUNCH(c, k_pad3, cdiv(B * N, 256), 256, 0, x, c0, B * N);
  float* dummy_style = c->alloc_n<float>((size_t)B * 4);      // never read: all style layers are constant
  LION_TRY(style_affine_all(f, dummy_style));
  LION_TRY(stat_pool_begin(f, (size_t)f.m->style_total * B * sizeof(double) + 4096));
  PF feat; feat.p = c0; feat.G = 1; feat.R = N;
  const float4* pts = c0;
  int n = N;
  for (size_t i = 0; i < e.sa.size(); ++i) {
    Level lv{pts, n};
    LION_TRY(sa_level_fwd(f, e.sa[i], lv, feat, (int)i));
    pts = lv.centers; n = lv.m;
  }
  float* pooled = c->alloc_n<float>((size_t)B * e.cfeat);
  LION_LAUNCH(c, k_max_rows, dim3(feat.G, B), 256, 0, feat.p, pooled, feat.G, n);
  LION_LAUNCH(c, k_small_linear, B, 128, e.cfeat * sizeof(float), e.mlp_w, e.mlp_b, pooled, e.cfeat, out, 2 * e.zdim, e.cfeat, 2 * e.zdim, 0);
  return check_launch(c, "style encoder");
}

// style -> (CLIP mixing, latent_points_ada.py:132-137) -> all 61 AdaGN style Linears in one launch; result in f.aff
static int unet_style_affine(Fwd& f, const float* style, const float* clip) {
  UnetBlk& u = *f.m->unet;
  Ctx* c = f.c;
  int B = f.B, E = u.embed_dim;
  if (u.clip) {
    if (!clip) { set_error("unet: this network needs clip_feat"); return LION_ERR_ARG; }
    float* cat = c->alloc_n<float>((size_t)B * (u.S + E));
    float* st2 = c->alloc_n<float>((size_t)B * u.S);
    if (!c->dry) LION_CHECK_CUDA(cudaMemcpy2DAsync(cat, (u.S + E) * sizeof(float), style, u.S * sizeof(float), u.S * sizeof(float), B, cudaMemcpyDeviceToDevice, c->stream));
    LION_LAUNCH(c, k_small_linear, B, 128, u.clip_dim * sizeof(float), u.cfw, u.cfb, clip, u.clip_dim, cat + u.S, u.S + E, u.clip_dim, E, 0);
    LION_LAUNCH(c, k_small_linear, B, 128, (u.S + E) * sizeof(float), u.scw, u.scb, cat, u.S + E, st2, u.S, u.S + E, u.S, 0);
    style = st2;
  }
  LION_TRY(check_launch(c, "unet style"));
  return style_affine_all(f, style);
}

// Everything of a U-Net forward that depends on coordinates (and t) only runs on the side stream, in this order: per SA
// level i its FPS and ball query, the time embedding after level 0, the voxel preps of level i + 1's points; then the
// FP stages' 3-NN searches from the deepest level up.  FPS alone is a chain of ~1360 latency-bound rounds on 32 SMs:
// there it hides under the first PVConvs.  The main stream waits for each result where it first needs it.
// Every buffer written on aux is allocated here, before the main stream's first mark(): no release() on the main
// stream can hand it to another buffer while aux may still be writing it.
static int unet_side_stream(Fwd& f, const float* t, float* temb, std::vector<Level>& L, cudaEvent_t& temb_done) {
  UnetBlk& u = *f.m->unet;
  Ctx* c = f.c;
  const int B = f.B, E = u.embed_dim, n_sa = (int)L.size();
  if (!c->dry) {
    LION_CHECK_CUDA(cudaEventRecord(u.aux_start, c->stream));
    LION_CHECK_CUDA(cudaStreamWaitEvent(c->aux, u.aux_start, 0));
    static DevOnce carve_once;
    if (carve_once.need()) {     // side-stream kernels share SMs with the convolutions: same (maximum) carve-out
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_ball_query_c4, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_three_nn_c4, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    }
  }
  for (int i = 0; i < n_sa; ++i) {
    const SABlk& sb = u.sa[i].back().sa;
    L[i].centers = c->alloc_n<float4>((size_t)B * sb.m);
    LION_TRY(sa_geometry(f, c->aux, sb, L[i], i));
    LION_TRY(record_on_aux(c, u.levels[i].sa_done, L[i].sa_done));
    if (i == 0 && temb) {
      // three tiny dependent launches (~45 us of latency) that nothing needs before level 1
      float* sinu = c->alloc_n<float>((size_t)B * E);
      float* h = c->alloc_n<float>((size_t)B * E);
      if (f.ur) { f.ur->a_sinu = sinu; f.ur->a_h = h; }
      LION_LAUNCH_ON(c, c->aux, k_time_sinusoid, B, 64, 0, t, u.d_freqs, sinu, E / 2, u.time_scale);
      LION_LAUNCH_ON(c, c->aux, k_small_linear, B, 128, E * sizeof(float), u.e0w, u.e0b, sinu, E, h, E, E, E, 1);
      LION_LAUNCH_ON(c, c->aux, k_small_linear, B, 128, E * sizeof(float), u.e2w, u.e2b, h, E, temb, E, E, E, 0);
      stamp(c, c->aux, "temb");
      LION_TRY(record_on_aux(c, u.temb_done, temb_done));
    }
    if (i + 1 == n_sa) continue;
    // the centres are level i + 1's points; voxelising them depends on coordinates only -- one CTA per shape, 13-25 us
    // each on the critical path otherwise
    Level& next = L[i + 1];
    next.pts = L[i].centers; next.n = sb.m;
    const std::vector<int>& rs = u.levels[i + 1].vox_r;
    for (int r : rs) { VoxPrep* vp; LION_TRY(get_vox(f, c->aux, next.pts, next.n, r, &vp)); }
    if (!rs.empty()) {
      stamp(c, c->aux, "voxprep", i + 1);
      LION_TRY(record_on_aux(c, u.levels[i + 1].vox_done, next.vox_done));
    }
  }
  for (int j = 0; j < (int)u.fp.size(); ++j) {
    const int l = n_sa - 1 - j;                     // FP stage j interpolates back onto level l's points
    LION_TRY(fp_geometry(f, c->aux, L[l], l));
    LION_TRY(record_on_aux(c, u.levels[l].nn_done, L[l].nn_done));
  }
  return 0;
}

static int unet_forward(Fwd& f, const float* x, const float* t, const float* style, const float* clip, float* out, int N) {
  UnetBlk& u = *f.m->unet;
  int B = f.B, E = u.embed_dim;
  Ctx* c = f.c;
  // time embedding: sinusoid -> Linear -> LeakyReLU(0.1) -> Linear  (latent_points_ada.py:53-57, :101-128), computed
  // on the side stream
  float* temb = nullptr;
  if (E > 0) {
    if (!t) { set_error("unet: this network needs timesteps"); return LION_ERR_ARG; }
    temb = c->alloc_n<float>((size_t)B * E);
  }
  // AdaGN style Linears (and the CLIP mixing in front of them) depend on the style only, which is constant over the
  // 1000 steps of a sampling run: style == nullptr means "use what lion_unet_cache_style computed"
  if (style) {
    LION_TRY(unet_style_affine(f, style, clip));
  } else {
    if (!f.m->aff_cache || f.m->aff_cache_B != B) { set_error("unet: no cached style for B=%d (call lion_unet_cache_style first)", B); return LION_ERR_STATE; }
    f.aff = f.m->aff_cache;
  }
  if (f.ur) LION_TRY(rec_copy(f, f.ur->aff, f.aff, sizeof(float) * B * f.m->style_total));
  LION_TRY(check_launch(c, "unet prologue"));
  LION_TRY(stat_pool_begin(f, (size_t)f.m->style_total * f.B * sizeof(double) + 4096));   // sum(2*C) doubles per shape

  const int n_sa = (int)u.sa.size();
  // level-0 inputs: coords = xyz, features = all input channels (the latent x[B,N,4] itself is a PF with G=1; a
  // 3-channel cloud x[B,N,3] (PointTransPVC) is padded to (x, y, z, 0), which serves as coordinates AND features)
  float4* c0 = c->alloc_n<float4>((size_t)B * N);
  PF feat; feat.G = 1; feat.R = N;
  if (u.extra == 0) {
    LION_LAUNCH(c, k_pad3, cdiv(B * N, 256), 256, 0, x, c0, B * N);
    feat.p = c0;
  } else {
    LION_LAUNCH(c, k_make_coords, cdiv(B * N, 256), 256, 0, (const float4*)x, c0, B * N);
    feat.p = (float4*)x;
  }
  std::vector<Level> L(n_sa);
  L[0].pts = c0; L[0].n = N;
  cudaEvent_t temb_done = nullptr;
  LION_TRY(unet_side_stream(f, t, temb, L, temb_done));
  stamp(c, c->stream, "start");
  auto with_temb = [&](PF src, PF* dstp) -> int {   // cat(features, temb expanded) (:145)
    LION_TRY(wait_once(c, temb_done));
    PF d = alloc_pf(f, src.G + E / 4, src.R);
    LION_LAUNCH(c, k_copy_groups, dim3(cdiv(src.R, 256), src.G, B), 256, 0, src.p, d.p, src.G, d.G, 0, src.R);
    LION_LAUNCH(c, k_fill_groups, dim3(cdiv(src.R, 256), E / 4, B), 256, 0, temb, E, d.p, d.G, src.G, src.R);
    *dstp = d;
    return check_launch(c, "concat temb");
  };
  // shared memory a convolution CTA may claim while side-stream kernels are resident on its SM (see conv_tc_run)
  constexpr int CONV_SMEM_BESIDE_AUX = 196 * 1024;
  for (int i = 0; i < n_sa; ++i) {
    c->conv_smem_cap = i == 0 ? CONV_SMEM_BESIDE_AUX : 0;      // the side stream is busy during level 0
    L[i].feat = feat;
    LION_TRY(wait_once(c, L[i].vox_done));
    if (i > 0 && temb) LION_TRY(with_temb(feat, &feat));
    LION_TRY(sa_level_fwd(f, u.sa[i], L[i], feat, i));
  }
  c->conv_smem_cap = 0;
  // skip features of level 0 are the extra channels only (inputs[:, 3:], :153): packed as
  // one group [f, 0, 0, 0]
  L[0].feat = u.extra == 1 ? alloc_pf(f, 1, N) : PF();
  if (u.extra == 1) LION_LAUNCH(c, k_extract_extra, cdiv(B * N, 256), 256, 0, (const float4*)x, L[0].feat.p, B * N);
  if (u.use_att) {
    PF o = alloc_pf(f, feat.G, feat.R);
    LION_TRY(attn_fwd(f, u.gatt, feat, o.p, o.G, 0));
    feat = o;
    stamp(c, c->stream, "global_att");
  }
  for (size_t j = 0; j < u.fp.size(); ++j) {
    Level& lv = L[n_sa - 1 - j];
    if (f.ur) f.ur->stage = (int)j;
    for (auto& blk : u.fp[j]) {
      if (blk.kind == LION_KIND_FP) {
        PF cf = feat;
        if (temb) LION_TRY(with_temb(feat, &cf));          // torch.cat([features, temb]) (:160)
        if (f.ur) LION_TRY(rec_copy(f, f.ur->fp[j].cf, cf.p, pf_bytes(f, cf)));
        PF o = alloc_pf(f, blk.fp.mlp.cout() / 4, lv.n);
        LION_TRY(fp_fwd(f, blk.fp, lv, cf, o.p, o.G, 0));
        feat = o;
        stamp(c, c->stream, "fp.module", (int)j);
      } else {
        PF o = alloc_pf(f, blk.pv.cout / 4, lv.n);
        LION_TRY(pvconv_fwd(f, blk.pv, feat, lv.pts, o.p, o.G, 0));
        feat = o;
        stamp(c, c->stream, "fp.pvconv", (int)j);
      }
    }
    if (f.ur) LION_TRY(rec_copy(f, f.ur->fp[j].out, feat.p, pf_bytes(f, feat)));
  }
  PF h = alloc_pf(f, 32, feat.R);
  MlpRecord cls_rec;
  if (f.ur) {
    LION_TRY(rec_copy(f, f.ur->feat, feat.p, pf_bytes(f, feat)));
    f.rec = &cls_rec;
  }
  LION_TRY(shared_mlp_fwd(f, u.cls0, feat, 1, h.p, 32, 0));
  if (f.ur) {
    f.rec = nullptr;
    UnetRecord& R = *f.ur;
    const size_t BC = (size_t)B * 128;
    LION_TRY(rec_copy(f, R.cls_raw, cls_rec.raw[0], pf_bytes(f, h)));
    LION_TRY(rec_copy(f, R.hc, h.p, pf_bytes(f, h)));
    if (R.cls_sums && !c->dry) {
      LION_CHECK_CUDA(cudaMemcpy2DAsync(R.cls_sums, sizeof(double) * 128, cls_rec.ssum[0], sizeof(double) * cls_rec.stat_stride[0],
                                        sizeof(double) * 128, B, cudaMemcpyDeviceToDevice, c->stream));
      LION_CHECK_CUDA(cudaMemcpy2DAsync(R.cls_sums + BC, sizeof(double) * 128, cls_rec.ssq[0], sizeof(double) * cls_rec.stat_stride[0],
                                        sizeof(double) * 128, B, cudaMemcpyDeviceToDevice, c->stream));
    }
    if (R.cls_aff) {
      LION_TRY(rec_copy(f, R.cls_aff, cls_rec.scale[0], sizeof(float) * BC));
      LION_TRY(rec_copy(f, R.cls_aff + BC, cls_rec.shift[0], sizeof(float) * BC));
    }
  }
  if (u.num_classes == 4) {
    LION_TRY(run_conv(f, u.cls2, h.p, h.G, (float4*)out, 1, nullptr, nullptr, geom_rows(feat.R)));
  } else {
    PF o4 = alloc_pf(f, (u.num_classes + 3) / 4, feat.R);
    LION_TRY(run_conv(f, u.cls2, h.p, h.G, o4.p, o4.G, nullptr, nullptr, geom_rows(feat.R)));
    LION_LAUNCH(c, k_pf_to_pm, dim3(cdiv(feat.R, 256), o4.G, B), 256, 0, o4.p, out, o4.G, u.num_classes, feat.R);
  }
  // never consumed by a one-level network: still join the side stream (every other result was waited for above)
  LION_TRY(wait_once(c, temb_done));
  if (f.ur && temb) {
    LION_TRY(rec_copy(f, f.ur->sinu, f.ur->a_sinu, sizeof(float) * B * E));
    LION_TRY(rec_copy(f, f.ur->h, f.ur->a_h, sizeof(float) * B * E));
    LION_TRY(rec_copy(f, f.ur->temb, temb, sizeof(float) * B * E));
  }
  stamp(c, c->stream, "end");
  return check_launch(c, "unet epilogue");
}


// run `body` twice: a dry pass measuring the arena, then (after growing it) the real pass
template <typename F>
static int two_pass(Model* m, void* stream, int B, F body) {
  Ctx* c = m->ctx;
  std::unique_lock<std::mutex> lock;
  if (c->mu) lock = std::unique_lock<std::mutex>(*c->mu);
  c->stream = (cudaStream_t)stream;
  for (int pass = 0; pass < 2; ++pass) {
    c->dry = (pass == 0);
    c->reset();
    Fwd f{c, m, B};
    int rc = body(f);
    if (rc) { c->dry = false; return rc; }
    if (pass == 0) {
      LION_TRY(ctx_reserve(c, c->peak));
      LION_TRY(ctx_reserve_zgrid(c, c->zgrid_need));
    }
  }
  return 0;
}

}  // namespace lion

// =====================================================================================
// C ABI
// =====================================================================================
using namespace lion;

struct LionCtx { Ctx c; std::mutex mu; };
struct LionModel { Model m; };

extern "C" int lion_version(void) { return 100; }
extern "C" const char* lion_last_error(void) { return get_error(); }

extern "C" int lion_ctx_create(int device, LionCtx** out) {
  LION_REQUIRE(out, "lion_ctx_create: null out");
  LION_CHECK_CUDA(cudaSetDevice(device));
  LionCtx* h = new LionCtx();
  h->c.device = device;
  h->c.mu = &h->mu;
  cudaDeviceProp prop;
  LION_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
  h->c.num_sms = prop.multiProcessorCount;
  h->c.l2_bytes = prop.l2CacheSize;
  LION_CHECK_CUDA(cudaStreamCreateWithFlags(&h->c.aux, cudaStreamNonBlocking));
  LION_CHECK_CUDA(cudaMalloc(&h->c.d_cls_count, sizeof(unsigned long long)));
  LION_CHECK_CUDA(cudaMemset(h->c.d_cls_count, 0, sizeof(unsigned long long)));
  { const char* e = getenv("LION_TIMELINE");
    if (e && atoi(e) != 0) LION_CHECK_CUDA(cudaMalloc(&h->c.d_stamps, LION_MAX_STAMPS * sizeof(unsigned long long))); }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("lion_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
    delete h;
    return LION_ERR_STATE;
  }
  *out = h;
  return 0;
}
extern "C" int lion_ctx_destroy(LionCtx* h) {
  if (!h) return 0;
  if (h->c.base) cudaFree(h->c.base);
  if (h->c.zgrid) cudaFree(h->c.zgrid);
  if (h->c.aux) cudaStreamDestroy(h->c.aux);
  if (h->c.d_stamps) cudaFree(h->c.d_stamps);
  if (h->c.d_cls_count) cudaFree(h->c.d_cls_count);
  delete h;
  return 0;
}
extern "C" int lion_ctx_last_launches(LionCtx* h) { return h ? h->c.launches : 0; }
extern "C" int lion_ctx_last_conv_group(LionCtx* h) { return h ? h->c.conv_group_blocks : 0; }
extern "C" int lion_ctx_last_conv_stage_taps(LionCtx* h) { return h ? h->c.conv_stage_taps : 0; }
extern "C" int lion_ctx_set_conv_whole_slabs(LionCtx* h, int on) {
  LION_REQUIRE(h, "lion_ctx_set_conv_whole_slabs: null context");
  h->c.conv_whole_slabs = on != 0;
  return 0;
}
extern "C" int lion_ctx_set_sparse_conv1_dense(LionCtx* h, int on) {
  LION_REQUIRE(h, "lion_ctx_set_sparse_conv1_dense: null context");
  h->c.sparse_conv1_dense = on != 0;
  return 0;
}
extern "C" int lion_ctx_set_conv2_class_mode(LionCtx* h, int mode) {
  LION_REQUIRE(h && mode >= 0 && mode <= 2, "lion_ctx_set_conv2_class_mode: null context or mode not 0-2");
  h->c.conv2_class_mode = mode;
  return 0;
}
extern "C" int lion_ctx_last_conv2_class_blocks(LionCtx* h, long long* flagged, long long* total) {
  LION_REQUIRE(h && flagged && total, "lion_ctx_last_conv2_class_blocks: null argument");
  unsigned long long n = 0;
  LION_CHECK_CUDA(cudaSetDevice(h->c.device));
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  LION_CHECK_CUDA(cudaMemcpy(&n, h->c.d_cls_count, sizeof(n), cudaMemcpyDeviceToHost));
  *flagged = (long long)n; *total = h->c.cls_blocks;
  return 0;
}
extern "C" unsigned lion_ctx_generation(LionCtx* h) { return h ? h->c.generation : 0; }
extern "C" int lion_ctx_timeline(LionCtx* h, unsigned long long* t_ns, char* names, int max_entries) {
  LION_REQUIRE(h && t_ns && names && max_entries >= 0, "lion_ctx_timeline: null argument");
  if (!h->c.d_stamps) { set_error("lion_ctx_timeline: the context was created without LION_TIMELINE=1"); return LION_ERR_STATE; }
  int n = h->c.n_stamps < max_entries ? h->c.n_stamps : max_entries;
  LION_CHECK_CUDA(cudaSetDevice(h->c.device));
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  LION_CHECK_CUDA(cudaMemcpy(t_ns, h->c.d_stamps, (size_t)n * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; ++i) memcpy(names + (size_t)i * 24, h->c.stamp_names[i], 24);
  return n;
}
extern "C" size_t lion_ctx_arena_bytes(LionCtx* h) { return h ? h->c.cap : 0; }
extern "C" size_t lion_workspace_bytes(LionCtx* h) { return h ? h->c.cap + h->c.zgrid_cap : 0; }

extern "C" int lion_model_create(LionCtx* ctx, int kind, const int* desc, int ndesc, const float* const* params,
                                 int nparams, LionModel** out) {
  LION_REQUIRE(ctx && out && (desc || ndesc == 0) && (params || nparams == 0), "lion_model_create: null argument");
  LION_CHECK_CUDA(cudaSetDevice(ctx->c.device));
  std::unique_ptr<LionModel> h(new LionModel());
  Model* m = &h->m;
  m->ctx = &ctx->c; m->kind = kind;
  m->desc.assign(desc, desc + ndesc);
  m->params.assign(params, params + nparams);
  for (int i = 0; i < nparams; ++i) LION_REQUIRE(params[i], "lion_model_create: parameter %d is null", i);
  Cursor cur{m->params.data(), nparams};
  const std::vector<int>& d = m->desc;
  auto need = [&](int n) { return (int)d.size() >= n; };
  switch (kind) {
    case LION_KIND_UNET: LION_TRY(build_unet(m, cur)); break;
    // style_dim == 0 selects the non-Ada blocks of models/pvcnn2.py (plain GroupNorm(8), no `emd` parameters, no style)
    case LION_KIND_PVCONV: {   // [cin, cout, r, attn, S]
      LION_REQUIRE(need(5), "pvconv descriptor: [cin, cout, r, attn, style_dim]");
      m->S = d[4] > 0 ? d[4] : 4;
      m->block.reset(new Block()); m->block->kind = kind;
      LION_TRY(make_pvconv(m, m->block->pv, cur, d[0], d[1], d[2], d[3] != 0, d[4] == 0));
      break;
    }
    case LION_KIND_SA: {       // [cfeat, m, radius_bits, k, S, n_mlp, mlp...]
      LION_REQUIRE(need(6) && need(6 + d[5]), "sa descriptor: [cfeat, m, radius_bits, k, style_dim, n, outs...]");
      m->S = d[4] > 0 ? d[4] : 4;
      m->block.reset(new Block()); m->block->kind = kind;
      LION_TRY(make_sa(m, m->block->sa, cur, d[0], d[1], bits_to_float(d[2]), d[3], std::vector<int>(d.begin() + 6, d.begin() + 6 + d[5]), d[4] == 0));
      break;
    }
    case LION_KIND_FP: {       // [cc, cp, S, n_mlp, mlp...]
      LION_REQUIRE(need(4) && need(4 + d[3]), "fp descriptor: [cc, cp, style_dim, n, outs...]");
      m->S = d[2];
      m->block.reset(new Block()); m->block->kind = kind;
      LION_TRY(make_fp(m, m->block->fp, cur, d[0], d[1], std::vector<int>(d.begin() + 4, d.begin() + 4 + d[3])));
      break;
    }
    case LION_KIND_ATTN: {     // [C, heads]
      LION_REQUIRE(need(2), "attention descriptor: [C, heads]");
      LION_REQUIRE(d[0] % 4 == 0, "attention: C must be a multiple of 4");
      m->attn.reset(new AttnBlk());
      LION_TRY(make_attn(m, *m->attn, cur, d[0], d[1]));
      break;
    }
    case LION_KIND_SHARED_MLP: {   // [cin, S, n, outs...]
      LION_REQUIRE(need(3) && need(3 + d[2]), "shared_mlp descriptor: [cin, style_dim, n, outs...]");
      m->S = d[1] > 0 ? d[1] : 4;
      m->mlp.reset(new SharedMLPBlk());
      LION_TRY(make_shared_mlp(m, *m->mlp, cur, d[0], ident_map(d[0]), std::vector<int>(d.begin() + 3, d.begin() + 3 + d[2]), d[1] == 0));
      break;
    }
    case LION_KIND_GLOBAL_PRIOR: LION_TRY(global_prior_build(m, cur)); break;
    case LION_KIND_STYLE_ENC: LION_TRY(build_style_enc(m, cur)); break;
    case LION_KIND_ADAGN: {        // [C, S]
      LION_REQUIRE(need(2), "adagn descriptor: [C, style_dim]");
      m->S = d[1];
      LION_TRY(make_adagn(m, m->gn_single, cur, d[0]));
      break;
    }
    case LION_KIND_CONV3D: {       // [cin, cout, r]
      LION_REQUIRE(need(3) && d[0] > 0 && d[1] > 0 && d[2] > 0 && d[2] <= 64, "conv3d descriptor: [cin, cout, r]");
      const float* w = cur.next(); const float* bi = cur.next();
      LION_REQUIRE(!cur.bad, "conv3d: parameters are [weight, bias]");
      LION_TRY(make_conv(m, m->conv_single, w, bi, 27, d[0], d[1], ident_map(d[0])));
      break;
    }
    default: LION_REQUIRE(false, "lion_model_create: unknown kind %d", kind);
  }
  LION_REQUIRE(!cur.bad && cur.i == cur.n, "lion_model_create(kind %d): %d parameters given, %d consumed", kind, cur.n, cur.i);
  if (!m->style_layers.empty()) {
    LION_TRY(m->dmalloc(&m->d_style_layers, m->style_layers.size()));
    LION_CHECK_CUDA(cudaMemcpy(m->d_style_layers, m->style_layers.data(), m->style_layers.size() * sizeof(StyleLayer), cudaMemcpyHostToDevice));
  }
  LION_TRY(run_repack(m));
  *out = h.release();
  return 0;
}
extern "C" int lion_model_destroy(LionModel* h) { delete h; return 0; }
extern "C" int lion_model_refresh(LionModel* h) {
  LION_REQUIRE(h, "lion_model_refresh: null model");
  std::unique_lock<std::mutex> lock;                     // (ensure_f16 may be appending FP16 packing steps)
  if (h->m.ctx->mu) lock = std::unique_lock<std::mutex>(*h->m.ctx->mu);
  LION_CHECK_CUDA(cudaSetDevice(h->m.ctx->device));
  return run_repack(&h->m);
}

extern "C" int lion_unet_forward(LionModel* h, const float* x, const float* t, const float* style, const float* clip,
                                 float* out, int B, int N, void* stream) {
  return lion_unet_forward_flags(h, x, t, style, clip, out, B, N, 0, stream);
}
extern "C" int lion_unet_forward_flags(LionModel* h, const float* x, const float* t, const float* style, const float* clip,
                                       float* out, int B, int N, int flags, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_UNET, "lion_unet_forward: not a unet model");
  LION_REQUIRE(x && out && B > 0 && N > 0 && (flags & ~LION_FWD_CONV_FP16) == 0, "lion_unet_forward: bad arguments");
  Model* m = &h->m;
  const bool f16 = (flags & LION_FWD_CONV_FP16) != 0;
  if (f16) LION_TRY(ensure_f16(m, stream));
  return two_pass(m, stream, B, [&](Fwd& f) { f.conv_f16 = f16; return unet_forward(f, x, t, style, clip, out, N); });
}

extern "C" int lion_style_encoder_forward(LionModel* h, const float* x, float* out, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_STYLE_ENC, "lion_style_encoder_forward: not a style-encoder model");
  LION_REQUIRE(x && out && B > 0 && N > 0, "lion_style_encoder_forward: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) { return style_enc_forward(f, x, out, N); });
}

// Hoists everything that depends on the style only out of the denoising loop (the reference recomputes the 61 AdaGN
// Linears and the CLIP mixing every step, models/adagn.py:59-61, latent_points_ada.py:132-137): computes them once
// into a buffer owned by the model; later lion_unet_forward calls with style == NULL use it.  Not capturable when the
// buffer has to grow (first call / larger B).
extern "C" int lion_unet_cache_style(LionModel* h, const float* style, const float* clip, int B, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_UNET, "lion_unet_cache_style: not a unet model");
  LION_REQUIRE(style && B > 0, "lion_unet_cache_style: bad arguments");
  Model* m = &h->m;
  if (m->aff_cache_B < B) {
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing((cudaStream_t)stream, &st);
    LION_REQUIRE(st == cudaStreamCaptureStatusNone, "lion_unet_cache_style: the cache must be sized outside stream capture");
    LION_CHECK_CUDA(cudaSetDevice(m->ctx->device));
    LION_CHECK_CUDA(cudaDeviceSynchronize());
    if (m->aff_cache) LION_CHECK_CUDA(cudaFree(m->aff_cache));
    m->aff_cache = nullptr; m->aff_cache_B = 0;
    LION_CHECK_CUDA(cudaMalloc((void**)&m->aff_cache, (size_t)B * m->style_total * sizeof(float) + 16));
  }
  m->aff_cache_B = B;
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    LION_TRY(unet_style_affine(f, style, clip));
    if (!f.c->dry) LION_CHECK_CUDA(cudaMemcpyAsync(m->aff_cache, f.aff, (size_t)B * m->style_total * sizeof(float), cudaMemcpyDeviceToDevice, f.c->stream));
    return 0;
  });
}

// ---- block-level entry points on the reference's channel-major layouts -------------------
namespace {
PF to_pf(Fwd& f, const float* src, int C, int R) {
  PF p = alloc_pf(f, (C + 3) / 4, R);
  LION_LAUNCH(f.c, k_cm_to_pf, dim3(cdiv(R, 256), p.G, f.B), 256, 0, src, p.p, C, p.G, R);
  return p;
}
void from_pf(Fwd& f, PF p, float* dst, int C) {
  LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(p.R, 256), p.G, f.B), 256, 0, p.p, dst, C, p.G, p.R);
}
float4* to_c4(Fwd& f, const float* src, int N) {
  float4* c = f.c->alloc_n<float4>((size_t)f.B * N);
  LION_LAUNCH(f.c, k_cm_to_c4, dim3(cdiv(N, 256), f.B), 256, 0, src, c, N);
  return c;
}
}  // namespace

extern "C" int lion_pvconv_fwd(LionModel* h, const float* features, const float* coords, const float* style, float* out,
                               int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_PVCONV, "lion_pvconv_fwd: not a pvconv model");
  LION_REQUIRE(features && coords && (style || h->m.desc[4] == 0) && out && B > 0 && N > 0, "lion_pvconv_fwd: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) {
    const PVConvBlk& p = m->block->pv;
    LION_TRY(style_affine_all(f, style ? style : f.c->alloc_n<float>((size_t)B * 4)));
    PF x = to_pf(f, features, m->desc[0], N);
    float4* c4 = to_c4(f, coords, N);
    PF o = alloc_pf(f, p.cout / 4, N);
    LION_TRY(pvconv_fwd(f, p, x, c4, o.p, o.G, 0));
    from_pf(f, o, out, p.cout);
    return check_launch(f.c, "lion_pvconv_fwd");
  });
}

extern "C" int lion_sa_module_fwd(LionModel* h, const float* features, const float* coords, const float* style,
                                  float* out_features, float* out_coords, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_SA, "lion_sa_module_fwd: not an SA model");
  LION_REQUIRE(features && coords && (style || h->m.desc[4] == 0) && out_features && out_coords && B > 0 && N > 0, "lion_sa_module_fwd: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) {
    const SABlk& s = m->block->sa;
    LION_TRY(style_affine_all(f, style ? style : f.c->alloc_n<float>((size_t)B * 4)));
    PF x = to_pf(f, features, s.cfeat, N);
    Level lv{to_c4(f, coords, N), N};
    lv.centers = f.c->alloc_n<float4>((size_t)B * s.m);
    PF o = alloc_pf(f, s.mlp.cout() / 4, s.m);
    LION_TRY(sa_geometry(f, f.c->stream, s, lv, 0));
    LION_TRY(sa_fwd(f, s, x, lv, o.p, o.G, 0));
    from_pf(f, o, out_features, s.mlp.cout());
    LION_LAUNCH(f.c, k_c4_to_cm, dim3(cdiv(s.m, 256), B), 256, 0, lv.centers, out_coords, s.m);
    return check_launch(f.c, "lion_sa_module_fwd");
  });
}

extern "C" int lion_fp_module_fwd(LionModel* h, const float* points_coords, const float* centers_coords,
                                  const float* centers_features, const float* points_features, const float* style,
                                  float* out, int B, int N, int M, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_FP, "lion_fp_module_fwd: not an FP model");
  LION_REQUIRE(points_coords && centers_coords && centers_features && style && out && B > 0 && N > 0 && M > 0, "lion_fp_module_fwd: bad arguments");
  Model* m = &h->m;
  LION_REQUIRE((m->block->fp.cp > 0) == (points_features != nullptr), "lion_fp_module_fwd: points_features presence does not match the module");
  return two_pass(m, stream, B, [&](Fwd& f) {
    const FPBlk& b = m->block->fp;
    LION_TRY(style_affine_all(f, style));
    Level lv{to_c4(f, points_coords, N), N};
    lv.centers = to_c4(f, centers_coords, M); lv.m = M;
    PF cf = to_pf(f, centers_features, b.cc, M);
    if (b.cp) lv.feat = to_pf(f, points_features, b.cp, N);
    PF o = alloc_pf(f, b.mlp.cout() / 4, N);
    LION_TRY(fp_geometry(f, f.c->stream, lv, 0));
    LION_TRY(fp_fwd(f, b, lv, cf, o.p, o.G, 0));
    from_pf(f, o, out, b.mlp.cout());
    return check_launch(f.c, "lion_fp_module_fwd");
  });
}

extern "C" int lion_linear_attention_fwd(LionModel* h, const float* x, float* out, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_ATTN, "lion_linear_attention_fwd: not an attention model");
  LION_REQUIRE(x && out && B > 0 && N > 0, "lion_linear_attention_fwd: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) {
    const AttnBlk& a = *m->attn;
    PF xi = to_pf(f, x, a.C, N);
    PF o = alloc_pf(f, a.C / 4, N);
    LION_TRY(attn_fwd(f, a, xi, o.p, o.G, 0));
    from_pf(f, o, out, a.C);
    return check_launch(f.c, "lion_linear_attention_fwd");
  });
}

extern "C" int lion_shared_mlp_fwd(LionModel* h, const float* x, const float* style, float* out, int B, int R, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_SHARED_MLP, "lion_shared_mlp_fwd: not a shared-mlp model");
  LION_REQUIRE(x && (style || h->m.desc[1] == 0) && out && B > 0 && R > 0, "lion_shared_mlp_fwd: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) {
    const SharedMLPBlk& s = *m->mlp;
    LION_TRY(style_affine_all(f, style ? style : f.c->alloc_n<float>((size_t)B * 4)));
    PF xi = to_pf(f, x, s.conv[0].cin_ref, R);
    PF o = alloc_pf(f, s.cout() / 4, R);
    LION_TRY(shared_mlp_fwd(f, s, xi, 1, o.p, o.G, 0));
    from_pf(f, o, out, s.cout());
    return check_launch(f.c, "lion_shared_mlp_fwd");
  });
}

// ---- stand-alone AdaGN / SE3d / Swish (reference interfaces models/adagn.py:45-65,
// models/pvcnn2_ada.py:27-41, :74-83); the fused path never calls these -------------------------
extern "C" int lion_adagn_fwd(LionModel* h, const float* x, const float* style, float* out, int B, int R, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_ADAGN, "lion_adagn_fwd: not an AdaGN model");
  LION_REQUIRE(x && style && out && B > 0 && R > 0, "lion_adagn_fwd: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) {
    const AdaGNW& g = m->gn_single;
    LION_TRY(style_affine_all(f, style));
    PF xi = to_pf(f, x, g.C, R);
    double *ssum, *ssq;
    LION_TRY(alloc_stats(f, g.C, &ssum, &ssq));
    LION_LAUNCH(f.c, k_row_stats, dim3(cdiv(R, 1024) > 64 ? 64 : cdiv(R, 1024), xi.G, B), 256, 0, xi.p, ssum, ssq, xi.G, R, g.C);
    AffSrc a;
    LION_TRY(run_affine(f, g, ssum, ssq, g.C, (double)R, nullptr, nullptr, a));
    PF o = alloc_pf(f, xi.G, R);
    LION_LAUNCH(f.c, k_act_rows<1>, dim3(cdiv(R, 256), xi.G, B), 256, 0, xi.p, o.p, a, xi.G, g.C, R, xi.G, 0, 2);
    from_pf(f, o, out, g.C);
    return check_launch(f.c, "lion_adagn_fwd");
  });
}
extern "C" int lion_se3d_fwd(LionCtx* ctx, const float* w1, const float* w2, const float* x, float* out, int B, int C, int V,
                             void* stream) {
  LION_REQUIRE(ctx && w1 && w2 && x && out && B > 0 && C > 0 && C % 8 == 0 && C <= 1024 && V > 0, "lion_se3d_fwd: bad arguments");
  Model tmp;
  tmp.ctx = &ctx->c;
  return two_pass(&tmp, stream, B, [&](Fwd& f) {
    PF xi = to_pf(f, x, C, V);
    double *ssum, *ssq;
    LION_TRY(alloc_stats(f, xi.G * 4, &ssum, &ssq));
    LION_LAUNCH(f.c, k_row_stats, dim3(cdiv(V, 1024) > 64 ? 64 : cdiv(V, 1024), xi.G, B), 256, 0, xi.p, ssum, ssq, xi.G, V, xi.G * 4);
    float* gate = f.c->alloc_n<float>((size_t)B * C);
    LION_LAUNCH(f.c, k_se_gate, B, C, (C + C / 8) * sizeof(float), ssum, xi.G * 4, w1, w2, gate, C, (double)V);
    size_t total = (size_t)B * C * V;
    LION_LAUNCH(f.c, k_scale_or_swish, (unsigned)cdivz(total, 256), 256, 0, x, gate, out, (size_t)V, total);
    return check_launch(f.c, "lion_se3d_fwd");
  });
}
extern "C" int lion_swish_fwd(const float* x, float* out, size_t n, void* stream) {
  LION_REQUIRE(x && out && n > 0, "lion_swish_fwd: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_scale_or_swish, (unsigned)cdivz(n, 256), 256, 0, x, (const float*)nullptr, out, (size_t)1, n);
  return check_launch(&c, "lion_swish_fwd");
}

// ---- stand-alone Conv3d 3x3x3 + fused GroupNorm statistics (reference: nn.Conv3d in
// models/pvcnn2_ada.py:211-222 followed by AdaGN's GroupNorm, models/adagn.py:36) -----------------
extern "C" int lion_conv3d_gn_fwd(LionModel* h, const float* x, float* out, double* gn_sum, double* gn_sqsum, int B, void* stream) {
  return lion_conv3d_gn_fwd_flags(h, x, out, gn_sum, gn_sqsum, B, 0, stream);
}
extern "C" int lion_conv3d_gn_fwd_flags(LionModel* h, const float* x, float* out, double* gn_sum, double* gn_sqsum, int B,
                                        int flags, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_CONV3D, "lion_conv3d_gn_fwd: not a conv3d model");
  LION_REQUIRE(x && out && B > 0 && ((gn_sum == nullptr) == (gn_sqsum == nullptr)) && (flags & ~LION_FWD_CONV_FP16) == 0,
               "lion_conv3d_gn_fwd: bad arguments");
  Model* m = &h->m;
  if (flags & LION_FWD_CONV_FP16) LION_TRY(ensure_f16(m, stream));
  // FP16 where the FP16 kernel serves the shape; otherwise exactly the TF32 call
  const bool f16 = (flags & LION_FWD_CONV_FP16) && m->conv_single.tc16.w;
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    const ConvW& w = m->conv_single;
    const int cin = m->desc[0], cout = m->desc[1], r = m->desc[2];
    const int Gin = w.cin_pad / (f16 ? 8 : 4), Gout = (cout + 3) / 4, rp = r + 2, V = r * r * r;
    const size_t P = (size_t)rp * rp * rp;
    float4* gi = alloc_vg(f, Gin, r);
    LION_TRY(memset_async(f.c, gi, 0, sizeof(float4) * (size_t)B * Gin * P));
    if (f16)
      LION_LAUNCH(f.c, k_cm_to_vg_h8, dim3(cdiv(V, 256), Gin, B), 256, 0, x, gi, cin, Gin, r);
    else
      LION_LAUNCH(f.c, k_cm_to_vg, dim3(cdiv(V, 256), Gin, B), 256, 0, x, gi, cin, Gin, r, 1);
    float4* go = alloc_vg(f, Gout, r);
    double *ssum = nullptr, *ssq = nullptr;
    if (gn_sum) LION_TRY(alloc_stats(f, w.cout_pad, &ssum, &ssq));
    LION_TRY(run_conv(f, w, gi, Gin, go, Gout, ssum, ssq, geom_grid(r), nullptr, f16));
    LION_LAUNCH(f.c, k_vg_to_cm, dim3(cdiv(V, 256), Gout, B), 256, 0, go, out, cout, Gout, r);
    if (gn_sum && !f.c->dry) {
      LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sum, sizeof(double) * cout, ssum, sizeof(double) * w.cout_pad, sizeof(double) * cout, B,
                                        cudaMemcpyDeviceToDevice, f.c->stream));
      LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sqsum, sizeof(double) * cout, ssq, sizeof(double) * w.cout_pad, sizeof(double) * cout, B,
                                        cudaMemcpyDeviceToDevice, f.c->stream));
    }
    return check_launch(f.c, "lion_conv3d_gn_fwd");
  });
}

// ---- stage probes: intermediate results of the product code that a module's output hides (tests only) -------------
// A PVConv's first convolution as pvconv_fwd runs it (voxel prep, scatter, dense or sparse convolution with its fused
// GroupNorm sums).  path: 0 = pvconv_fwd's choice, 1 = dense, 2 = sparse; *path_taken = 1 or 2.
extern "C" int lion_pvconv_conv1_probe(LionModel* h, const float* features, const float* coords, int path, float* out,
                                       double* gn_sum, double* gn_sqsum, int* path_taken, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_PVCONV, "lion_pvconv_conv1_probe: not a pvconv model");
  LION_REQUIRE(features && coords && out && gn_sum && gn_sqsum && path >= 0 && path <= 2 && B > 0 && N > 0,
               "lion_pvconv_conv1_probe: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    const PVConvBlk& p = m->block->pv;
    const int r = p.r, rp = r + 2, P = rp * rp * rp, Gout = p.cout / 4;
    PF x = to_pf(f, features, m->desc[0], N);
    float4* c4 = to_c4(f, coords, N);
    VoxPrep* vp;
    LION_TRY(get_vox(f, f.c->stream, c4, N, r, &vp));
    Conv1Out c1;
    LION_TRY(pvconv_conv1(f, p, x, vp, path, true, c1, [] { return 0; }));
    // the dense path scattered into the context's zero grid: zero those voxels again (k_act_grid's extra blocks alone)
    if (!c1.sparse)
      LION_LAUNCH(f.c, k_act_grid<false>, dim3(cdiv(N, 256), Gout, B), 256, 0, c1.raw, nullptr, AffSrc{}, Gout, p.cout, rp, P, 0,
                  vp->ppos, c1.g_in, p.cin / 4, N, nullptr, nullptr);
    LION_LAUNCH(f.c, k_vg_to_cm, dim3(cdiv(r * r * r, 256), Gout, B), 256, 0, c1.raw, out, p.cout, Gout, r);
    if (!f.c->dry) {
      LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sum, sizeof(double) * p.cout, c1.ssum, sizeof(double) * p.c1.cout_pad,
                                        sizeof(double) * p.cout, B, cudaMemcpyDeviceToDevice, f.c->stream));
      LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sqsum, sizeof(double) * p.cout, c1.ssq, sizeof(double) * p.c1.cout_pad,
                                        sizeof(double) * p.cout, B, cudaMemcpyDeviceToDevice, f.c->stream));
      if (path_taken) *path_taken = c1.sparse ? 2 : 1;
    }
    return check_launch(f.c, "lion_pvconv_conv1_probe");
  });
}

// The sparse first convolution's vgrid and activity mask (include/lion_b200.h)
extern "C" int lion_pvconv_conv1_mask_probe(LionModel* h, const float* features, const float* coords, int* vgrid, unsigned* mask,
                                            int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_PVCONV, "lion_pvconv_conv1_mask_probe: not a pvconv model");
  LION_REQUIRE(features && coords && vgrid && mask && B > 0 && N > 0, "lion_pvconv_conv1_mask_probe: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    const PVConvBlk& p = m->block->pv;
    const int r = p.r, rp = r + 2, P = rp * rp * rp;
    PF x = to_pf(f, features, m->desc[0], N);
    float4* c4 = to_c4(f, coords, N);
    VoxPrep* vp;
    LION_TRY(get_vox(f, f.c->stream, c4, N, r, &vp));
    Conv1Out c1;
    LION_TRY(pvconv_conv1(f, p, x, vp, 2, false, c1, [] { return 0; }));
    LION_TRY(memcpy_d2d(f.c, vgrid, vp->vgrid, sizeof(int) * (size_t)B * P));
    LION_TRY(memcpy_d2d(f.c, mask, c1.mask, sizeof(unsigned) * (size_t)B * cdiv(r * r * r, 32)));
    return check_launch(f.c, "lion_pvconv_conv1_mask_probe");
  });
}

// An SA module's MLP as sa_fwd runs it.  path: 0 = sa_fwd's choice, 1 = unfused kernels, 2 = fused; *path_taken = 1 or 2.
// Per layer l (C_l channels, offsets o_l = B * (C_0 + ... + C_{l-1})): gn_sum / gn_sqsum [B][C_l] doubles and the folded
// AdaGN scale / shift [B][C_l] at o_l; pool_mm [B][C_last/4][M][2][4] = per (centre, channel) minimum and maximum of the
// last layer's pre-activation over the 32 neighbours; centers [B,3,M].
extern "C" int lion_sa_mlp_probe(LionModel* h, const float* features, const float* coords, const float* style, int path,
                                 float* centers, double* gn_sum, double* gn_sqsum, float* scale, float* shift, float* pool_mm,
                                 int* path_taken, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_SA, "lion_sa_mlp_probe: not an SA model");
  LION_REQUIRE(features && coords && (style || h->m.desc[4] == 0) && centers && gn_sum && gn_sqsum && scale && shift && pool_mm &&
               path >= 0 && path <= 2 && B > 0 && N > 0, "lion_sa_mlp_probe: bad arguments");
  Model* m = &h->m;
  const SABlk& s = m->block->sa;
  LION_REQUIRE((int)s.mlp.conv.size() <= MLP_REC_MAX, "lion_sa_mlp_probe: more than %d layers", MLP_REC_MAX);
  LION_REQUIRE(path != 2 || sa_fused_usable(s), "lion_sa_mlp_probe: the fused kernels do not serve this module");
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    MlpRecord rec;
    rec.force = path;
    f.rec = &rec;
    LION_TRY(style_affine_all(f, style ? style : f.c->alloc_n<float>((size_t)B * 4)));
    PF x = to_pf(f, features, s.cfeat, N);
    Level lv{to_c4(f, coords, N), N};
    lv.centers = f.c->alloc_n<float4>((size_t)B * s.m);
    PF o = alloc_pf(f, s.mlp.cout() / 4, s.m);
    LION_TRY(sa_geometry(f, f.c->stream, s, lv, 0));
    LION_TRY(sa_fwd(f, s, x, lv, o.p, o.G, 0));
    if (rec.n != (int)s.mlp.conv.size() || !rec.pool_mm) {
      set_error("lion_sa_mlp_probe: the last layer does not run the pooled epilogue");
      return LION_ERR_ARG;
    }
    if (!f.c->dry) {
      // (the arena sa_fwd released is not reused before these copies: they are the next work on the stream)
      size_t off = 0;
      for (int l = 0; l < rec.n; ++l) {
        const int C = s.mlp.conv[l].cout;
        LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sum + off, sizeof(double) * C, rec.ssum[l], sizeof(double) * rec.stat_stride[l],
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sqsum + off, sizeof(double) * C, rec.ssq[l], sizeof(double) * rec.stat_stride[l],
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpyAsync(scale + off, rec.scale[l], sizeof(float) * B * C, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpyAsync(shift + off, rec.shift[l], sizeof(float) * B * C, cudaMemcpyDeviceToDevice, f.c->stream));
        off += (size_t)B * C;
      }
      LION_CHECK_CUDA(cudaMemcpyAsync(pool_mm, rec.pool_mm, sizeof(float) * B * s.mlp.cout() * s.m * 2, cudaMemcpyDeviceToDevice,
                                      f.c->stream));
      if (path_taken) *path_taken = rec.fused ? 2 : 1;
    }
    LION_LAUNCH(f.c, k_c4_to_cm, dim3(cdiv(s.m, 256), B), 256, 0, lv.centers, centers, s.m);
    return check_launch(f.c, "lion_sa_mlp_probe");
  });
}

// A whole PVConv as lion_pvconv_fwd runs it, with the intermediate results of its second half (C = cout, V = r^3):
// raw1 / raw2 [B,C,r,r,r] the two convolutions' raw outputs; act1 [B,C,r+2,r+2,r+2] the AdaGN-1 + Swish grid conv2
// reads, halo included; rawp [B,C,N] the point branch's raw 1x1 output; sums [4][B][C] doubles: conv2's sum and sum of
// squares, then the point branch's; affine [6][B][C]: scale / shift of AdaGN-1, of the point-branch AdaGN and of AdaGN-2
// with the SE gate multiplied in; fused [B,C,N] devoxelised + point branch (the attention's input; without attention
// the module output); out [B,C,N]; *conv2_kernel (may be NULL) = 0 SIMT, 1 row tiles, 2 / 4 interior-block groups.
extern "C" int lion_pvconv_probe(LionModel* h, const float* features, const float* coords, const float* style, float* raw1,
                                 float* act1, float* raw2, float* rawp, double* sums, float* affine, float* fused, float* out,
                                 int* conv2_kernel, int B, int N, void* stream) {
  return lion_pvconv_probe_flags(h, features, coords, style, raw1, act1, raw2, rawp, sums, affine, fused, out, conv2_kernel, B, N,
                                 0, stream);
}
// flags LION_FWD_CONV_FP16: act1 is the FP16 grid (where the FP16 kernel serves conv2), returned widened to fp32
extern "C" int lion_pvconv_probe_flags(LionModel* h, const float* features, const float* coords, const float* style, float* raw1,
                                       float* act1, float* raw2, float* rawp, double* sums, float* affine, float* fused, float* out,
                                       int* conv2_kernel, int B, int N, int flags, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_PVCONV, "lion_pvconv_probe: not a pvconv model");
  LION_REQUIRE(features && coords && (style || h->m.desc[4] == 0) && raw1 && act1 && raw2 && rawp && sums && affine && fused &&
               out && B > 0 && N > 0 && (flags & ~LION_FWD_CONV_FP16) == 0, "lion_pvconv_probe: bad arguments");
  Model* m = &h->m;
  const bool f16 = (flags & LION_FWD_CONV_FP16) != 0;
  if (f16) LION_TRY(ensure_f16(m, stream));
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    const PVConvBlk& p = m->block->pv;
    const int C = p.cout, G = C / 4, r = p.r, rp = r + 2;
    PvRecord rec;
    f.pv = &rec;
    f.conv_f16 = f16;
    LION_TRY(style_affine_all(f, style ? style : f.c->alloc_n<float>((size_t)B * 4)));
    PF x = to_pf(f, features, m->desc[0], N);
    float4* c4 = to_c4(f, coords, N);
    PF o = alloc_pf(f, G, N);
    LION_TRY(pvconv_fwd(f, p, x, c4, o.p, o.G, 0));
    // (the arena pvconv_fwd released is not reused before these copies: they are the next work on the stream)
    LION_LAUNCH(f.c, k_vg_to_cm, dim3(cdiv(r * r * r, 256), G, B), 256, 0, rec.raw1, raw1, C, G, r);
    if (rec.act1_f16)
      LION_LAUNCH(f.c, k_h8_to_cm, dim3(cdiv(rp * rp * rp, 256), G / 2, B), 256, 0, rec.act1, act1, C, G / 2, rp * rp * rp);
    else
      LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(rp * rp * rp, 256), G, B), 256, 0, rec.act1, act1, C, G, rp * rp * rp);
    LION_LAUNCH(f.c, k_vg_to_cm, dim3(cdiv(r * r * r, 256), G, B), 256, 0, rec.raw2, raw2, C, G, r);
    LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), G, B), 256, 0, rec.rawp, rawp, C, G, N);
    LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), G, B), 256, 0, rec.fused, fused, C, G, N);
    from_pf(f, o, out, C);
    if (!f.c->dry) {
      const size_t BC = (size_t)B * C;
      const AffSrc* st[2] = {&rec.a2, &rec.ap};
      for (int k = 0; k < 2; ++k) {
        LION_CHECK_CUDA(cudaMemcpy2DAsync(sums + (2 * k) * BC, sizeof(double) * C, st[k]->ssum, sizeof(double) * st[k]->stat_stride,
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpy2DAsync(sums + (2 * k + 1) * BC, sizeof(double) * C, st[k]->ssq, sizeof(double) * st[k]->stat_stride,
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
      }
      const AffSrc* af[3] = {&rec.a1, &rec.ap, &rec.a2};
      for (int k = 0; k < 3; ++k) {
        LION_CHECK_CUDA(cudaMemcpyAsync(affine + (2 * k) * BC, af[k]->scale, sizeof(float) * BC, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpyAsync(affine + (2 * k + 1) * BC, af[k]->shift, sizeof(float) * BC, cudaMemcpyDeviceToDevice, f.c->stream));
      }
      if (conv2_kernel) *conv2_kernel = rec.conv2;
    }
    return check_launch(f.c, "lion_pvconv_probe");
  });
}

// A linear attention as lion_linear_attention_fwd runs it: qkv [B, 3 H 32, N] (q, k, v of every head), o [B, H 32, N]
// the output before the projection, out [B,C,N].
extern "C" int lion_attention_probe(LionModel* h, const float* x, float* qkv, float* o, float* out, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_ATTN, "lion_attention_probe: not an attention model");
  LION_REQUIRE(x && qkv && o && out && B > 0 && N > 0, "lion_attention_probe: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    const AttnBlk& a = *m->attn;
    const int hid = a.heads * 32;
    PvRecord rec;
    f.pv = &rec;
    PF xi = to_pf(f, x, a.C, N);
    PF y = alloc_pf(f, a.C / 4, N);
    LION_TRY(attn_fwd(f, a, xi, y.p, y.G, 0));
    LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), 3 * hid / 4, B), 256, 0, rec.qkv, qkv, 3 * hid, 3 * hid / 4, N);
    LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), hid / 4, B), 256, 0, rec.o, o, hid, hid / 4, N);
    from_pf(f, y, out, a.C);
    return check_launch(f.c, "lion_attention_probe");
  });
}

// [B][N][3] 32-bit words -> [B][3][N]: the 3-NN indices or weights in the reference's layout
__global__ void k_nn_to_cm(const unsigned* __restrict__ src, unsigned* __restrict__ dst, int N) {
  int b = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  for (int k = 0; k < 3; ++k) dst[((size_t)b * 3 + k) * N + j] = src[((size_t)b * N + j) * 3 + k];
}

// An FP module as lion_fp_module_fwd runs it: nn_idx / nn_wgt [B,3,N] the 3-NN; cat [B, cc + roundup(cp,4), N] the MLP
// input, padding channels included (NaN-filled before its producers run); per layer l (C_l channels): raw / act
// [B,C_l,N] at offset B N (C_0 + ... + C_{l-1}) the raw 1x1 output and the activated output (the last is the module
// output), gn_sum / gn_sqsum (doubles) and the folded scale / shift [B,C_l] at offset B (C_0 + ... + C_{l-1}).
extern "C" int lion_fp_probe(LionModel* h, const float* points_coords, const float* centers_coords, const float* centers_features,
                             const float* points_features, const float* style, int* nn_idx, float* nn_wgt, float* cat, float* raw,
                             float* act, double* gn_sum, double* gn_sqsum, float* scale, float* shift, int B, int N, int M,
                             void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_FP, "lion_fp_probe: not an FP model");
  LION_REQUIRE(points_coords && centers_coords && centers_features && style && nn_idx && nn_wgt && cat && raw && act && gn_sum &&
               gn_sqsum && scale && shift && B > 0 && N > 0 && M > 0, "lion_fp_probe: bad arguments");
  Model* m = &h->m;
  const FPBlk& b = m->block->fp;
  LION_REQUIRE((b.cp > 0) == (points_features != nullptr), "lion_fp_probe: points_features presence does not match the module");
  LION_REQUIRE((int)b.mlp.conv.size() <= MLP_REC_MAX, "lion_fp_probe: more than %d layers", MLP_REC_MAX);
  return two_pass(m, stream, B, [&](Fwd& f) -> int {
    MlpRecord rec;
    f.rec = &rec;
    LION_TRY(style_affine_all(f, style));
    Level lv{to_c4(f, points_coords, N), N};
    lv.centers = to_c4(f, centers_coords, M); lv.m = M;
    PF cf = to_pf(f, centers_features, b.cc, M);
    if (b.cp) lv.feat = to_pf(f, points_features, b.cp, N);
    PF o = alloc_pf(f, b.mlp.cout() / 4, N);
    LION_TRY(fp_geometry(f, f.c->stream, lv, 0));
    LION_TRY(fp_fwd(f, b, lv, cf, o.p, o.G, 0));
    // (the arena fp_fwd released is not reused before these copies: they are the next work on the stream)
    LION_LAUNCH(f.c, k_nn_to_cm, dim3(cdiv(N, 256), B), 256, 0, (const unsigned*)lv.nn_idx, (unsigned*)nn_idx, N);
    LION_LAUNCH(f.c, k_nn_to_cm, dim3(cdiv(N, 256), B), 256, 0, (const unsigned*)lv.nn_wgt, (unsigned*)nn_wgt, N);
    const int Gcat = b.mlp.cin_pad / 4;
    LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), Gcat, B), 256, 0, rec.cat, cat, 4 * Gcat, Gcat, N);
    size_t off = 0;
    for (int l = 0; l < (int)b.mlp.conv.size(); ++l) {
      const int C = b.mlp.conv[l].cout, G = C / 4;
      if (l >= rec.n || !rec.raw[l] || !rec.act[l] || rec.act_G[l] != G || rec.act_off[l] != 0) {
        set_error("lion_fp_probe: layer %d was not recorded", l);
        return LION_ERR_STATE;
      }
      LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), G, B), 256, 0, rec.raw[l], raw + off * N, C, G, N);
      LION_LAUNCH(f.c, k_pf_to_cm, dim3(cdiv(N, 256), G, B), 256, 0, rec.act[l], act + off * N, C, G, N);
      if (!f.c->dry) {
        LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sum + off, sizeof(double) * C, rec.ssum[l], sizeof(double) * rec.stat_stride[l],
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpy2DAsync(gn_sqsum + off, sizeof(double) * C, rec.ssq[l], sizeof(double) * rec.stat_stride[l],
                                          sizeof(double) * C, B, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpyAsync(scale + off, rec.scale[l], sizeof(float) * B * C, cudaMemcpyDeviceToDevice, f.c->stream));
        LION_CHECK_CUDA(cudaMemcpyAsync(shift + off, rec.shift[l], sizeof(float) * B * C, cudaMemcpyDeviceToDevice, f.c->stream));
      }
      off += (size_t)B * C;
    }
    return check_launch(f.c, "lion_fp_probe");
  });
}

// A U-Net forward as lion_unet_forward runs it, with its glue recorded.  taps: 4 + 6 n_fp + 5 device pointers, any of
// them NULL (not recorded), in this order (PF = packed [B][G][R][4], G = ceil(C / 4)):
//   sinu, h, temb [B][E]: the sinusoid, after the first Linear + LeakyReLU, the time embedding;
//   aff [B][style_total]: every AdaGN (factor | bias) vector, as computed (style != NULL) or cached (style == NULL);
//   per FP stage j: cf PF [C_in + E, M] the centre features after the time-embedding concat; nn_idx (int) / nn_wgt
//   [B][N][3] the 3-NN of the level's points; skip PF [roundup(cp,4), N] the level's skip features (not written when
//   cp = 0); cat PF [cc + roundup(cp,4), N] the MLP input (NaN-filled before its producers run); out PF [C_j, N] the
//   stage's output after its PVConvs;
//   head: feat PF [C, N] its input; cls_raw PF [128, N] cls0's raw output; cls_sums [2][B][128] (doubles) its
//   GroupNorm sums; cls_aff [2][B][128] its folded scale / shift; hc PF [128, N] its output.
// style_table [n_style][2] (host): (out_off, n_out) of every AdaGN style Linear in build order.
extern "C" int lion_unet_probe(LionModel* h, const float* x, const float* t, const float* style, const float* clip, float* out,
                               void* const* taps, int ntaps, int* style_table, int n_style, int B, int N, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_UNET, "lion_unet_probe: not a unet model");
  LION_REQUIRE(x && out && taps && B > 0 && N > 0, "lion_unet_probe: bad arguments");
  Model* m = &h->m;
  const int n_fp = (int)m->unet->fp.size();
  LION_REQUIRE(n_fp <= UNET_REC_FP, "lion_unet_probe: more than %d FP stages", UNET_REC_FP);
  LION_REQUIRE(ntaps == 4 + 6 * n_fp + 5, "lion_unet_probe: %d taps given, %d expected", ntaps, 4 + 6 * n_fp + 5);
  LION_REQUIRE(n_style == (int)m->style_layers.size(), "lion_unet_probe: %d style layers expected, the network has %d", n_style,
               (int)m->style_layers.size());
  for (int i = 0; style_table && i < n_style; ++i) {
    style_table[2 * i] = m->style_layers[i].out_off;
    style_table[2 * i + 1] = m->style_layers[i].n_out;
  }
  UnetRecord rec;
  int k = 0;
  auto tap = [&]() { return (float*)taps[k++]; };
  rec.sinu = tap(); rec.h = tap(); rec.temb = tap(); rec.aff = tap();
  for (int j = 0; j < n_fp; ++j) {
    UnetRecord::Stage& s = rec.fp[j];
    s.cf = tap(); s.nn_idx = (int*)tap(); s.nn_wgt = tap(); s.skip = tap(); s.cat = tap(); s.out = tap();
  }
  rec.feat = tap(); rec.cls_raw = tap(); rec.cls_sums = (double*)tap(); rec.cls_aff = tap(); rec.hc = tap();
  return two_pass(m, stream, B, [&](Fwd& f) { f.ur = &rec; return unet_forward(f, x, t, style, clip, out, N); });
}

extern "C" int lion_global_prior_step(LionModel* h, const float* x, const float* t, const float* clip, float* out, int B,
                                      void* stream) {
  return lion_global_prior_forward(h, x, t, clip, out, B, stream);
}

extern "C" int lion_global_prior_forward(LionModel* h, const float* x, const float* t, const float* clip, float* out,
                                         int B, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_GLOBAL_PRIOR, "lion_global_prior_forward: not a global-prior model");
  LION_REQUIRE(x && t && out && B > 0, "lion_global_prior_forward: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) { (void)f; return global_prior_forward(m, x, t, clip, out, B); });
}

// A global-prior forward as lion_global_prior_forward runs it, with every Linear's output copied out.  taps: 5 + 4 ncell
// device pointers [B][width] fp32, any of them NULL: pe [emb], t0 [4 emb], temb [nf], cmap [nf] (CLIP models only), h0
// [nf], then per cell a [nf], bb [nf], s [nf/8], h [nf].
extern "C" int lion_global_prior_probe(LionModel* h, const float* x, const float* t, const float* clip, float* out,
                                       void* const* taps, int ntaps, int B, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_GLOBAL_PRIOR, "lion_global_prior_probe: not a global-prior model");
  LION_REQUIRE(x && t && out && taps && B > 0, "lion_global_prior_probe: bad arguments");
  Model* m = &h->m;
  const int ncell = m->desc[3], has_clip = m->desc[4];    // desc: [D, nf, emb, ncell, clip, clip_dim, scale_bits]
  LION_REQUIRE(ntaps == 5 + 4 * ncell, "lion_global_prior_probe: %d taps given, %d expected", ntaps, 5 + 4 * ncell);
  LION_REQUIRE(has_clip || !taps[3], "lion_global_prior_probe: a cmap tap for a network without CLIP");
  GpRecord rec;
  std::vector<GpRecord::Cell> cells(ncell);
  int k = 0;
  auto tap = [&]() { return (float*)taps[k++]; };
  rec.pe = tap(); rec.t0 = tap(); rec.temb = tap(); rec.cmap = tap(); rec.h0 = tap();
  for (GpRecord::Cell& cl : cells) { cl.a = tap(); cl.bb = tap(); cl.s = tap(); cl.h = tap(); }
  rec.cells = cells.data();
  return two_pass(m, stream, B, [&](Fwd& f) { (void)f; return global_prior_forward(m, x, t, clip, out, B, &rec); });
}

extern "C" size_t lion_global_prior_saved_floats(LionModel* h, int B) {
  if (!h || h->m.kind != LION_KIND_GLOBAL_PRIOR || B <= 0) return 0;
  return global_prior_saved_floats(&h->m, B);
}

extern "C" int lion_global_prior_forward_train(LionModel* h, const float* x, const float* t, const float* clip,
                                               const float* drop_mask, float* saved, float* out, int B, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_GLOBAL_PRIOR, "lion_global_prior_forward_train: not a global-prior model");
  LION_REQUIRE(x && t && saved && out && B > 0, "lion_global_prior_forward_train: bad arguments");
  Model* m = &h->m;
  return two_pass(m, stream, B, [&](Fwd& f) { (void)f; return global_prior_forward_train(m, x, t, clip, drop_mask, saved, out, B); });
}

extern "C" int lion_global_prior_backward(LionModel* h, const float* saved, const float* clip, const float* drop_mask,
                                          const float* gout, float* gx, float* const* gparams, int nparams, int B,
                                          void* stream) {
  return lion_global_prior_backward_probe(h, saved, clip, drop_mask, gout, gx, gparams, nparams, nullptr, 0, B, stream);
}

// The backward as lion_global_prior_backward runs it, with the gradients between the Linears copied out.  taps: 4 + 5 ncell
// device pointers [B][width] fp32, any of them NULL: gtemb [nf], gt0 [4 emb], gcmap [nf] (CLIP models only), gh0 [nf],
// then per cell gh [nf], gz [nf], gs [nf/8], gbb [nf], gz1 [nf].
extern "C" int lion_global_prior_backward_probe(LionModel* h, const float* saved, const float* clip, const float* drop_mask,
                                                const float* gout, float* gx, float* const* gparams, int nparams,
                                                void* const* taps, int ntaps, int B, void* stream) {
  LION_REQUIRE(h && h->m.kind == LION_KIND_GLOBAL_PRIOR, "lion_global_prior_backward: not a global-prior model");
  LION_REQUIRE(saved && gout && gx && gparams && B > 0, "lion_global_prior_backward: bad arguments");
  for (int i = 0; i < nparams; ++i) LION_REQUIRE(gparams[i], "lion_global_prior_backward: gradient %d is null", i);
  Model* m = &h->m;
  const int ncell = m->desc[3], has_clip = m->desc[4];
  GpBwdRecord rec;
  std::vector<GpBwdRecord::Cell> cells(ncell);
  if (taps) {
    LION_REQUIRE(ntaps == 4 + 5 * ncell, "lion_global_prior_backward_probe: %d taps given, %d expected", ntaps, 4 + 5 * ncell);
    LION_REQUIRE(has_clip || !taps[2], "lion_global_prior_backward_probe: a gcmap tap for a network without CLIP");
    int k = 0;
    auto tap = [&]() { return (float*)taps[k++]; };
    rec.gtemb = tap(); rec.gt0 = tap(); rec.gcmap = tap(); rec.gh0 = tap();
    for (GpBwdRecord::Cell& cl : cells) { cl.gh = tap(); cl.gz = tap(); cl.gs = tap(); cl.gbb = tap(); cl.gz1 = tap(); }
    rec.cells = cells.data();
  }
  return two_pass(m, stream, B, [&](Fwd& f) {
    (void)f;
    return global_prior_backward(m, saved, clip, drop_mask, gout, gx, (const float* const*)gparams, nparams, B,
                                 taps ? &rec : nullptr);
  });
}

// ---- measurement hook: time the convolution kernel alone (bench.py roofline leg) ------------
__global__ void k_fill_pattern(float* p, size_t n, float scale) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { unsigned h = (unsigned)(i * 2654435761u) ^ 0x9e3779b9u; h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
               p[i] = scale * ((float)(h & 0xffff) / 32768.0f - 1.0f); }
}
extern "C" int lion_bench_conv(LionCtx* ctx, int ntaps, int cin, int cout, int r_or_rows, int B, int iters, int warmup,
                               float* ms_out, double* flops_out, void* stream) {
  LION_REQUIRE(ctx && ms_out && flops_out && (ntaps == 27 || ntaps == 1) && cin % 4 == 0 && cout % 8 == 0 && B > 0 && iters > 0,
               "lion_bench_conv: bad arguments");
  LION_CHECK_CUDA(cudaSetDevice(ctx->c.device));
  LionModel h;
  Model* m = &h.m;
  m->ctx = &ctx->c;
  float *wref = nullptr, *bref = nullptr;
  size_t nw = (size_t)cout * cin * ntaps;
  LION_TRY(m->dmalloc(&wref, nw));
  LION_TRY(m->dmalloc(&bref, (size_t)cout));
  k_fill_pattern<<<(unsigned)cdivz(nw, 256), 256>>>(wref, nw, 0.05f);
  k_fill_pattern<<<cdiv(cout, 256), 256>>>(bref, cout, 0.1f);
  ConvW w;
  LION_TRY(make_conv(m, w, wref, bref, ntaps, cin, cout, ident_map(cin)));
  LION_TRY(run_repack(m));
  ConvGeom geo = ntaps == 27 ? geom_grid(r_or_rows) : geom_rows(r_or_rows);
  size_t guard = ntaps == 27 ? (size_t)(r_or_rows + 2) * (r_or_rows + 2) + (r_or_rows + 2) + 8 : 256;
  size_t n_in = (size_t)B * (cin / 4) * geo.rows + 2 * guard, n_out = (size_t)B * (cout / 4) * geo.rows + 2 * guard;
  float4 *din = nullptr, *dout = nullptr;
  double* stats = nullptr;
  LION_TRY(m->dmalloc(&din, n_in));
  LION_TRY(m->dmalloc(&dout, n_out));
  LION_TRY(m->dmalloc(&stats, (size_t)2 * B * w.cout_pad));
  k_fill_pattern<<<(unsigned)cdivz(n_in * 4, 256), 256>>>((float*)din, n_in * 4, 1.0f);
  LION_CHECK_CUDA(cudaMemset(stats, 0, sizeof(double) * 2 * B * w.cout_pad));
  LION_CHECK_CUDA(cudaDeviceSynchronize());
  Ctx* c = &ctx->c;
  c->stream = (cudaStream_t)stream;
  c->dry = false;
  Fwd f{c, m, B};
  cudaEvent_t e0, e1;
  LION_CHECK_CUDA(cudaEventCreate(&e0));
  LION_CHECK_CUDA(cudaEventCreate(&e1));
  for (int i = 0; i < warmup; ++i)
    LION_TRY(run_conv(f, w, din + guard, cin / 4, dout + guard, cout / 4, stats, stats + (size_t)B * w.cout_pad, geo));
  LION_CHECK_CUDA(cudaEventRecord(e0, c->stream));
  for (int i = 0; i < iters; ++i)
    LION_TRY(run_conv(f, w, din + guard, cin / 4, dout + guard, cout / 4, stats, stats + (size_t)B * w.cout_pad, geo));
  LION_CHECK_CUDA(cudaEventRecord(e1, c->stream));
  LION_CHECK_CUDA(cudaEventSynchronize(e1));
  float ms = 0;
  LION_CHECK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *ms_out = ms / iters;
  // algorithmic FLOPs of the dense convolution (interior voxels / rows only, no halo work counted)
  double rows = ntaps == 27 ? (double)r_or_rows * r_or_rows * r_or_rows : (double)r_or_rows;
  *flops_out = 2.0 * B * rows * ntaps * (double)cin * cout;
  return 0;
}

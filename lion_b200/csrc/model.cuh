// lion_b200 -- host-side model description shared by net.cu, conv_tc.cu and global_prior.cu.
#pragma once
#include <functional>
#include <memory>
#include <vector>
#include "common.cuh"

namespace lion {

struct StyleLayer { const float* w; const float* b; int n_out; int out_off; };

// tensor-core packing of a convolution's weights and the tiling it is packed for (conv_tc_prepare);
// w == nullptr -> SIMT kernel only
struct ConvTcW {
  float* w = nullptr;    // [n-tile][chunk][tap group][tap][KG][NT][4], tf32-rounded (tc16: [...][NT][8] fp16 bits)
  int NT = 0;            // output channels per CTA (wgmma N, <= 128)
  int KG = 0;            // 16-byte input groups (4 fp32 / 8 fp16 channels) per pipeline chunk (2, 4 or 8)
  int nchunk = 0;        // chunks
  int ntg = 0, tpg = 0;  // tap groups (x planes) and taps per group: (3, 9) or (1, 1)
};

struct Cursor {
  const float* const* p;
  int n, i = 0;
  bool bad = false;
  const float* next() {
    if (i >= n) { bad = true; return nullptr; }
    return p[i++];
  }
};

struct ConvW {
  int ntaps = 1, cin_ref = 0, cin_pad = 0, cout = 0, cout_pad = 0;
  float* wt = nullptr;      // [ntaps][cin_pad][cout_pad]   (SIMT kernel)
  float* bias = nullptr;    // [cout_pad]
  ConvTcW tc;               // tensor-core packing (conv_tc.cuh); tc.w == nullptr when unsupported
  ConvTcW tc16;             // FP16 packing and tiling (conv_tc_prepare_f16, made on the first FP16 forward) or w == nullptr
};
struct AdaGNW {
  const float* gamma = nullptr; const float* beta = nullptr;
  int C = 0; int style_off = 0;
};

struct Model;
struct Fwd;

struct SharedMLPBlk {
  std::vector<ConvW> conv;
  std::vector<AdaGNW> gn;
  int cin_pad = 0;
  int cout() const { return conv.back().cout; }
};
struct AttnBlk {
  ConvW qkv, out;
  int C = 0, heads = 0;
};
struct PVConvBlk {
  int cin = 0, cout = 0, r = 0;
  ConvW c1, c2;
  ConvW c1y;            // sparse first convolution: 1x1 "convolution" x[v] -> y[v][tap][cout] (c1y.tc.w set when available)
  AdaGNW g1, g2;
  const float* se1 = nullptr; const float* se2 = nullptr;
  SharedMLPBlk point;
  bool has_attn = false;
  AttnBlk attn;
};
struct SABlk {
  int cfeat = 0, m = 0, k = 0;
  float radius = 0;
  SharedMLPBlk mlp;
};
struct FPBlk {
  int cc = 0, cp = 0;   // interpolated channels, skip channels
  SharedMLPBlk mlp;
};
struct Block {
  int kind;   // LION_KIND_PVCONV / SA / FP
  PVConvBlk pv; SABlk sa; FPBlk fp;
};
// Point level l of the U-Net: the input points of SA level l, which FP stage n_sa - 1 - l interpolates back onto.
// What the side stream prepares for it (unet_forward) is fixed by the architecture and decided at build time.
struct UnetLevel {
  std::vector<int> vox_r;   // distinct PVConv resolutions on these points: the SA level's first, then the FP stage's
  cudaEvent_t sa_done = nullptr, vox_done = nullptr, nn_done = nullptr;   // FPS + ball query, voxel preps, 3-NN
};
struct UnetBlk {
  int num_classes, embed_dim, extra, input_dim, use_att, clip, clip_dim, S;
  const float *e0w = nullptr, *e0b = nullptr, *e2w = nullptr, *e2b = nullptr;
  const float *cfw = nullptr, *cfb = nullptr, *scw = nullptr, *scb = nullptr;
  float* d_freqs = nullptr;
  float time_scale = 1.0f;                                // sde.embedding_scale: t is scaled before the sinusoid
  std::vector<std::vector<Block>> sa, fp;
  std::vector<UnetLevel> levels;                          // [n_sa]
  cudaEvent_t aux_start = nullptr, temb_done = nullptr;   // the side stream may start; the time embedding is done
  AttnBlk gatt;
  SharedMLPBlk cls0;
  ConvW cls2;
};
// PointNetPlusEncoder (models/shapelatent_modules.py:13-52): SA levels on the non-Ada blocks, max over points, Linear
struct StyleEncBlk {
  int input_dim = 3, zdim = 128, cfeat = 0;
  std::vector<std::vector<Block>> sa;
  const float* mlp_w = nullptr; const float* mlp_b = nullptr;
};
struct GlobalPriorBlk;   // global_prior.cu
// Caller buffers (device, [B][width] fp32) that lion_global_prior_probe has global_prior_forward fill, each copied on
// the stream right after the Linear that produced it (real pass only; never set in a product call).  Any may be null.
struct GpRecord {
  float *pe = nullptr, *t0 = nullptr, *temb = nullptr, *cmap = nullptr, *h0 = nullptr;   // [emb], [4 emb], [nf] x 3
  // conv1 + ReLU (+ dropout), conv2 + ReLU [nf]; SE fc0 + ReLU [nf/8]; cell output [nf]; SE gate sigmoid(fc2) [nf]
  // (gate: written by the reduce itself, not copied, and only by the training forward)
  struct Cell { float *a, *bb, *s, *h, *gate; };
  const Cell* cells = nullptr;               // one per cell
};
// Caller buffers ([B][width] fp32) that lion_global_prior_backward_probe has global_prior_backward fill with the
// gradients flowing between the Linears.  Any may be null.
struct GpBwdRecord {
  float *gtemb = nullptr, *gt0 = nullptr, *gcmap = nullptr, *gh0 = nullptr;   // [nf], [4 emb], [nf], [nf]
  // d/d(cell output) [nf]; d/d(fc2 pre-sigmoid) [nf]; d/d(fc0 pre-ReLU) [nf/8]; d/d(conv2 pre-ReLU) [nf];
  // d/d(conv1 pre-ReLU) [nf]
  struct Cell { float *gh, *gz, *gs, *gbb, *gz1; };
  const Cell* cells = nullptr;
};
int global_prior_build(Model* m, Cursor& cur);
int global_prior_forward(Model* m, const float* x, const float* t, const float* clip, float* out, int B,
                         const GpRecord* rec = nullptr, const float* drop = nullptr);
size_t global_prior_saved_floats(const Model* m, int B);
int global_prior_forward_train(Model* m, const float* x, const float* t, const float* clip, const float* drop,
                               float* saved, float* out, int B);
int global_prior_backward(Model* m, const float* saved, const float* clip, const float* drop, const float* gout,
                          float* gx, const float* const* gparams, int nparams, int B, const GpBwdRecord* rec = nullptr);
void global_prior_free(GlobalPriorBlk*);

struct Model {
  Ctx* ctx = nullptr;
  int kind = 0;
  std::vector<int> desc;
  std::vector<const float*> params;
  std::vector<void*> owned;
  std::vector<cudaEvent_t> events;
  // Launches that derive the packed weights from the parameters, in order (a step may read an earlier one's output).
  // Run once at build and again by lion_model_refresh after the parameters changed in place.  A step captures device
  // pointers and sizes by value: the ConvWs it serves live in vectors that may still grow while the model is built.
  std::vector<std::function<void()>> repack;
  bool f16_ready = false;      // the FP16 packings exist (ensure_f16 in net.cu)
  std::vector<StyleLayer> style_layers;
  StyleLayer* d_style_layers = nullptr;
  int style_total = 0;
  int S = 128;
  float* aff_cache = nullptr;  // [aff_cache_B][style_total]: the AdaGN style Linears of a step-invariant style (lion_unet_cache_style)
  int aff_cache_B = 0;
  std::unique_ptr<UnetBlk> unet;
  std::unique_ptr<Block> block;
  std::unique_ptr<AttnBlk> attn;
  std::unique_ptr<SharedMLPBlk> mlp;
  std::unique_ptr<StyleEncBlk> senc;
  GlobalPriorBlk* gp = nullptr;
  AdaGNW gn_single;            // LION_KIND_ADAGN
  ConvW conv_single;           // LION_KIND_CONV3D

  template <typename T> int dmalloc(T** p, size_t n) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 16);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e)); return LION_ERR_OOM; }
    owned.push_back(q);
    *p = (T*)q;
    return 0;
  }
  int make_event(cudaEvent_t* e) {
    cudaError_t r = cudaEventCreateWithFlags(e, cudaEventDisableTiming);
    if (r != cudaSuccess) { set_error("cudaEventCreate failed: %s", cudaGetErrorString(r)); return LION_ERR_CUDA; }
    events.push_back(*e);
    return 0;
  }
  ~Model() {
    for (void* q : owned) cudaFree(q);
    for (cudaEvent_t e : events) cudaEventDestroy(e);
    if (aff_cache) cudaFree(aff_cache);
    if (gp) global_prior_free(gp);
  }
};


int make_conv(Model* m, ConvW& w, const float* w_src, const float* b_src, int ntaps, int cin_ref, int cout,
              const std::vector<int>& kmap);
std::vector<int> ident_map(int c);
static inline int roundup(int a, int b) { return (a + b - 1) / b * b; }

// geometry of one convolution launch (rows, tap offsets, halo mask)
struct ConvGeom {
  int ntaps;
  int off[27];
  int rp;        // r+2 for a VG, 0 for a PF (no halo mask)
  int rows;      // rows per (b, group): P or R
  int p_begin, p_end;
  const unsigned char* occ;   // optional 64-row occupancy flags of the INPUT ([B][occ_stride]); null = dense
  int occ_stride;
  // optional class-valued 64-row blocks of a 3x3x3 row-tile convolution's output and their values (conv_tc.cu:
  // Params::cls_flag); cls_store: store those rows too
  const unsigned char* cls_flag;
  int cls_stride;
  const float4* cls;
  bool cls_store;
};

// conv_tc.cu
int conv_tc_prepare(Model* m, ConvW& w);
int conv_tc_prepare_f16(Model* m, ConvW& w);
bool conv_tc_usable(const ConvW& w, const ConvGeom& geo);
bool conv_tc_row_tiles_3x3(const ConvW& w);
// sparse first convolution, GEMM half (sparse_conv.cu)
bool ygemm_usable(const ConvW& y);
int ygemm_run(Ctx* c, const ConvW& y, const float4* xc, float* out, int ld, const int* nocc, int B, int N);
// fused set-abstraction MLP (sa_fused.cu)
bool sa_fused_usable(const SABlk& s);
int sa_fused_run(Ctx* c, const SABlk& s, const float4* feat, const float4* points, const float4* centers, const int* nidx,
                 const float* scale1, const float* shift1, double* ssum, double* ssq, int stat_stride, float* pool_mm,
                 int B, int N);
int conv_tc_run(Ctx* c, const ConvW& w, const float4* in, int Gin, float4* out, int Gout_store, double* ssum,
                double* ssq, const ConvGeom& geo, int B, float* pool_mm = nullptr, bool f16 = false);

}  // namespace lion

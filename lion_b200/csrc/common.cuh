// lion_b200 -- shared plumbing for the sm_90a kernels: error reporting, the per-context
// bump arena (no allocation inside a forward), launch helpers, small device utilities.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <string>
#include <vector>
#include <mutex>

namespace lion {

// ---------------------------------------------------------------------------------------
// errors: every C-ABI entry returns 0 / negative code and never exits the process
// (the reference's kernels exit(-1), third_party/pvcnn/functional/src/cuda_utils.cuh:28-37).
// ---------------------------------------------------------------------------------------
enum : int { LION_OK = 0, LION_ERR_CUDA = -1, LION_ERR_ARG = -2, LION_ERR_OOM = -3, LION_ERR_STATE = -4 };

void set_error(const char* fmt, ...);
const char* get_error();

#define LION_CHECK_CUDA(expr)                                                          \
  do {                                                                                 \
    cudaError_t _e = (expr);                                                           \
    if (_e != cudaSuccess) {                                                           \
      lion::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return lion::LION_ERR_CUDA;                                                      \
    }                                                                                  \
  } while (0)

#define LION_REQUIRE(cond, ...)                                                        \
  do {                                                                                 \
    if (!(cond)) {                                                                     \
      lion::set_error(__VA_ARGS__);                                                    \
      return lion::LION_ERR_ARG;                                                       \
    }                                                                                  \
  } while (0)

#define LION_TRY(expr)                                                                 \
  do {                                                                                 \
    int _r = (expr);                                                                   \
    if (_r != 0) return _r;                                                            \
  } while (0)

// ---------------------------------------------------------------------------------------
// Context: device, stream of the current call, bump arena.
// A forward is run twice: a dry pass (no launches) that measures the arena high-water mark,
// then -- after growing the arena if needed, outside any graph capture -- the real pass.
// ---------------------------------------------------------------------------------------
constexpr int LION_MAX_STAMPS = 256;
struct Ctx {
  int device = 0;
  int num_sms = 132;
  int l2_bytes = 50 << 20;
  cudaStream_t stream = nullptr;
  cudaStream_t aux = nullptr;     // side stream for work that is independent of the main chain (FPS, neighbour searches)
  char* base = nullptr;      // arena
  char* zgrid = nullptr;     // persistent all-zero voxel grid (scatter target; re-zeroed after use)
  size_t zgrid_cap = 0, zgrid_need = 0;
  size_t cap = 0;
  size_t off = 0;
  size_t peak = 0;
  unsigned generation = 0;   // bumped whenever the arena / zero grid moves: graphs captured before are stale
  std::mutex* mu = nullptr;  // one forward at a time per context (ctypes releases the GIL); owned by LionCtx
  bool dry = false;
  int launches = 0;          // kernels launched by the last real pass (gpu_launches evidence)
  // > 0 while side-stream kernels (FPS, neighbour searches) are expected in flight: persistent convolution CTAs then
  // leave this much shared memory unclaimed so that both can be resident on one SM (see conv_tc_run)
  int conv_smem_cap = 0;
  // blocks per group of the last tensor-core convolution on interior blocks (2 or 4; 0 when it ran on row tiles)
  int conv_group_blocks = 0;
  // taps per weight stage of the last tensor-core convolution: 9 (whole 3x3x3 slabs), 3 (slabs in 3-tap parts) or 1 (1x1)
  int conv_stage_taps = 0;
  // set by tests only (lion_ctx_set_conv_whole_slabs): 3x3x3 weight slabs are always streamed whole
  bool conv_whole_slabs = false;
  // set by tests only (lion_ctx_set_sparse_conv1_dense): the sparse first convolution stores every voxel of its output
  // and the activation pass reads every interior position (no activity mask)
  bool sparse_conv1_dense = false;
  // set by tests only (lion_ctx_set_conv2_class_mode): 0 = the second convolution of a PVConv whose first one ran sparse
  // skips its class-valued blocks, 1 = it computes every block, 2 = it skips them and its output grid is filled with NaNs
  // first (no reader may touch an unstored row)
  int conv2_class_mode = 0;
  unsigned long long* d_cls_count = nullptr;   // class-valued blocks flagged by the last k_conv2_flags (device)
  long long cls_blocks = 0;                    // the blocks it examined
  // LION_TIMELINE=1 (diagnostic, tools/timeline_step.py): %globaltimer stamps dropped into both streams at block
  // boundaries -- this image has no nsys, and a step's critical path across the two streams is not visible otherwise
  unsigned long long* d_stamps = nullptr;
  int n_stamps = 0;
  char stamp_names[LION_MAX_STAMPS][24];

  void reset() { off = 0; peak = 0; launches = 0; zgrid_need = 0; n_stamps = 0; }
  // 256-byte aligned sub-allocation; in dry mode returns a fake non-null pointer.
  void* alloc(size_t bytes) {
    size_t a = (off + 255) & ~size_t(255);
    off = a + bytes;
    if (off > peak) peak = off;
    if (dry) return (void*)(uintptr_t)(0x1000 + a);
    return base + a;
  }
  template <typename T> T* alloc_n(size_t n) { return (T*)alloc(n * sizeof(T)); }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};

int ctx_reserve(Ctx* c, size_t bytes);   // grow arena (sync; not capturable)

// launch helpers of a forward: skipped in dry mode, counted in Ctx::launches.  LION_LAUNCH uses the context's stream,
// LION_LAUNCH_ON the given one (the side stream).
#define LION_LAUNCH_ON(ctx, stream, kernel, grid, block, smem, ...)                    \
  do {                                                                                 \
    if (!(ctx)->dry) {                                                                 \
      kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__);                      \
      (ctx)->launches++;                                                               \
    }                                                                                  \
  } while (0)
#define LION_LAUNCH(ctx, kernel, grid, block, smem, ...) LION_LAUNCH_ON(ctx, (ctx)->stream, kernel, grid, block, smem, __VA_ARGS__)

static __global__ void k_stamp(unsigned long long* p) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  *p = t;
}
// stamps on the side stream are named "aux:<name>"
inline void stamp(Ctx* c, cudaStream_t s, const char* name, int idx = -1) {
  if (!c->d_stamps || c->dry || c->n_stamps >= LION_MAX_STAMPS) return;
  const char* pre = s == c->aux ? "aux:" : "";
  if (idx >= 0) snprintf(c->stamp_names[c->n_stamps], 24, "%s%s%d", pre, name, idx);
  else snprintf(c->stamp_names[c->n_stamps], 24, "%s%s", pre, name);
  k_stamp<<<1, 1, 0, s>>>(c->d_stamps + c->n_stamps);
  c->n_stamps++;
}

inline int memset_async(Ctx* c, void* p, int v, size_t bytes, cudaStream_t s) {
  if (c->dry || bytes == 0) return 0;
  LION_CHECK_CUDA(cudaMemsetAsync(p, v, bytes, s));
  return 0;
}
inline int memset_async(Ctx* c, void* p, int v, size_t bytes) { return memset_async(c, p, v, bytes, c->stream); }
inline int memcpy_d2d(Ctx* c, void* d, const void* s, size_t bytes) {
  if (c->dry || bytes == 0) return 0;
  LION_CHECK_CUDA(cudaMemcpyAsync(d, s, bytes, cudaMemcpyDeviceToDevice, c->stream));
  return 0;
}
inline int check_launch(Ctx* c, const char* what) {
  if (c->dry) return 0;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("kernel launch failed in %s: %s", what, cudaGetErrorString(e));
    return LION_ERR_CUDA;
  }
  return 0;
}

// "opt this kernel into > 48 KB of dynamic shared memory" is a PER-DEVICE attribute: a process-wide once-flag would
// skip the opt-in on the second GPU of a multi-device process.  DevOnce keeps one flag per device ordinal.
struct DevOnce {
  unsigned long long done[4] = {0, 0, 0, 0};     // 256 device ordinals
  bool need() {
    int d = 0;
    if (cudaGetDevice(&d) != cudaSuccess || d < 0 || d >= 256) return true;
    unsigned long long bit = 1ull << (d & 63);
    if (done[d >> 6] & bit) return false;
    done[d >> 6] |= bit;
    return true;
  }
};

static inline int cdiv(int a, int b) { return (a + b - 1) / b; }
static inline size_t cdivz(size_t a, size_t b) { return (a + b - 1) / b; }

// ---------------------------------------------------------------------------------------
// device utilities
// ---------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// x * sigmoid(x).  __fdividef (MUFU.RCP + multiply, <= 2 ulp) instead of an IEEE division (~10 instructions with its slow
// path): the activation passes run at ~1 float4 per clock per SM and are instruction-bound otherwise.  For x < -87 the
// denominator overflows and the quotient is -0 (the exact value underflows as well).
__device__ __forceinline__ float swishf(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
__device__ __forceinline__ float4 f4_affine(float4 v, float4 s, float4 t) {
  return make_float4(fmaf(v.x, s.x, t.x), fmaf(v.y, s.y, t.y), fmaf(v.z, s.z, t.z), fmaf(v.w, s.w, t.w));
}
__device__ __forceinline__ float4 f4_swish(float4 v) {
  return make_float4(swishf(v.x), swishf(v.y), swishf(v.z), swishf(v.w));
}
// round-to-nearest(-away) to TF32, the unbiased conversion cuDNN applies to tensor-core operands;
// used where the ONLY consumer of a tensor is a wgmma tf32 convolution (which would
// otherwise truncate the low 13 mantissa bits, a one-sided error that accumulates over layers)
__device__ __forceinline__ float tf32_rna(float x) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
  return __uint_as_float(u);
}
__device__ __forceinline__ float4 f4_tf32(float4 v) { return make_float4(tf32_rna(v.x), tf32_rna(v.y), tf32_rna(v.z), tf32_rna(v.w)); }
// squared distance with the FMA contraction nvcc applies to the reference's
// dx*dx + dy*dy + dz*dz (t = dy*dy; t = fma(dx,dx,t); t = fma(dz,dz,t)); see oracle/point_ops.py.
__device__ __forceinline__ float sqdist_ref(float dx, float dy, float dz) {
  return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
}
#endif

}  // namespace lion

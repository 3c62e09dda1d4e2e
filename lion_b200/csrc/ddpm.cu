// lion_b200 -- the per-step update of the ancestral DDPM sampler, one elementwise kernel.
//
// Reference: utils/diffusion_pvd.py:283-296 (noise, mean, x update) with
// get_q_posterior_mean :475-486 and get_p_log_scales :155-168.  The reference evaluates, in
// fp32 tensor ops on 0-dim scalars (SURVEY.md Appendix B 13a):
//   t > 0:  mean = (1/sqrt(alpha_t)) * (x - (beta_t * eps) / sqrt(1 - abar_t))
//           x'   = mean + exp(0.5*log(beta_t)) * z * temp
//   t = 0:  x'   = (1/sqrt(abar_0)) * (x - sqrt(1 - abar_0) * eps)
// The per-step scalars come from a device table row selected by a device-side step counter,
// so the captured step graph is replayed without host-side parameter updates.
//   table row t: { c0, c1, c2, c3 } =
//     t > 0: { 1/sqrt(alpha_t), beta_t, sqrt(1-abar_t), exp(0.5*log beta_t) }
//     t = 0: { 1/sqrt(abar_0),  sqrt(1-abar_0), 1, 0 }   (flagged by c3 == 0 and t == 0)
// and the same operation order is replayed (no FMA contraction).
#include "common.cuh"
#include "../../include/lion_b200.h"

namespace lion {

__global__ void k_ddpm_update(const float* x /* may alias xo (in-place update) */, const float* __restrict__ eps, const float* __restrict__ noise,
                              float* xo, const float4* __restrict__ tables, const int* __restrict__ step,
                              float temp, size_t n, float* __restrict__ hist, int T) {
  int t = *step;
  float4 c = tables[t];
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float xv = x[i], e = eps[i];
  float r;
  if (t == 0) {
    r = __fmul_rn(c.x, __fsub_rn(xv, __fmul_rn(c.y, e)));
  } else {
    float mean = __fmul_rn(c.x, __fsub_rn(xv, __fdiv_rn(__fmul_rn(c.y, e), c.z)));
    r = __fadd_rn(mean, __fmul_rn(__fmul_rn(c.w, noise[i]), temp));
  }
  xo[i] = r;
  if (hist) hist[(size_t)(T - 1 - t) * n + i] = r;   // trajectory slot of this step (pred_x)
}

// Row `*step` of a device-resident noise block [rows][n] -> dst[n].  Lets a caller who supplies every step's noise
// (given_noise: host noise uploaded ahead of the loop) keep the copy INSIDE the captured step graph, selected by the same
// device-side step counter as the update's table row: no per-step host work besides the graph replay.
__global__ void k_ddpm_fetch_noise(float4* __restrict__ dst, const float4* __restrict__ block, const int* __restrict__ step, size_t n4) {
  const int t = *step;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n4) dst[i] = block[(size_t)t * n4 + i];
}

__global__ void k_ddpm_set_step(int* step, float* t_out, int B, int t_index, int advance) {
  int t = advance ? (*step - 1) : t_index;
  __syncthreads();
  if (threadIdx.x == 0) *step = t;
  for (int b = threadIdx.x; b < B; b += blockDim.x) t_out[b] = (float)(t + 1);
}

// DDIM update (reference: utils/diffusion_pvd.py:450-465):  x = x_noisy * a;  x += c*eps + sigma*z
// with the 0-dim fp32 scalars a = sqrt(abar_next/abar_t), c, sigma of step i (host-built table
// row { a, c, sigma, t+1 }, see DiffusionDiscretized._ddim_tables); same operation order, no FMA.
// noise is the whole [S][n] block of the run's draws; row i is consumed at step i.
__global__ void k_ddim_update(const float* x /* may alias xo (in-place update) */, const float* __restrict__ eps, const float* __restrict__ noise,
                              float* xo, const float4* __restrict__ tables, const int* __restrict__ step,
                              size_t n, float* __restrict__ hist) {
  int s = *step;
  float4 c = tables[s];
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float z = noise ? noise[(size_t)s * n + i] : 0.0f;
  float r = __fadd_rn(__fmul_rn(x[i], c.x), __fadd_rn(__fmul_rn(c.y, eps[i]), __fmul_rn(c.z, z)));
  xo[i] = r;
  if (hist) hist[(size_t)s * n + i] = r;
}

// step index i -> i+1 (or set), and the model's timestep vector t_out[b] = tables[i].w
__global__ void k_ddim_set_step(int* step, float* t_out, const float4* __restrict__ tables, int B, int S, int index, int advance) {
  int s = advance ? (*step + 1) : index;
  __syncthreads();
  if (threadIdx.x == 0) *step = s;
  float t = s < S ? tables[s].w : 0.0f;
  for (int b = threadIdx.x; b < B; b += blockDim.x) t_out[b] = t;
}

// diffusers-style DDPMScheduler.step (the models/lion.py:37-80 route; algorithm of diffusers 0.11.1,
// scheduling_ddpm.py, epsilon prediction, clip_sample=False):
//   x0   = (x - sqrt(1-abar_t) * eps) / sqrt(abar_t)
//   prev = c0 * x0 + c1 * x,   c0 = sqrt(abar_{t-1}) * beta_t / (1-abar_t),  c1 = sqrt(alpha_t) * (1-abar_{t-1}) / (1-abar_t)
//   x'   = prev + sqrt(var_t) * z   for t > 0,   x' = prev   at t = 0
// table row t (8 floats): { sqrt(1-abar_t), sqrt(abar_t), c0, c1, sqrt(var_t), 0, 0, 0 }.
__global__ void k_sched_step(const float* x /* may alias xo (in-place update) */, const float* __restrict__ eps, const float* __restrict__ noise,
                             float* xo, const float4* __restrict__ tables, const int* __restrict__ step, size_t n) {
  int t = *step;
  float4 c = tables[2 * t];
  float sigma = tables[2 * t + 1].x;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float xv = x[i];
  float x0 = __fdiv_rn(__fsub_rn(xv, __fmul_rn(c.x, eps[i])), c.y);
  float prev = __fadd_rn(__fmul_rn(c.z, x0), __fmul_rn(c.w, xv));
  xo[i] = t > 0 ? __fadd_rn(prev, __fmul_rn(sigma, noise[i])) : prev;
}

}  // namespace lion

using namespace lion;

extern "C" int lion_ddpm_update(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                                const int* step_ptr, float temp, size_t n, float* hist, int T, void* stream) {
  LION_REQUIRE(x && eps && x_out && tables && step_ptr && n > 0, "lion_ddpm_update: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddpm_update, (unsigned)cdivz(n, 256), 256, 0, x, eps, noise ? noise : x, x_out, (const float4*)tables, step_ptr, temp, n, hist, T);
  return check_launch(&c, "lion_ddpm_update");
}
extern "C" int lion_ddpm_fetch_noise(float* dst, const float* block, const int* step_ptr, size_t n, void* stream) {
  LION_REQUIRE(dst && block && step_ptr && n > 0 && n % 4 == 0, "lion_ddpm_fetch_noise: bad arguments (n must be a multiple of 4)");
  LION_REQUIRE(((uintptr_t)dst | (uintptr_t)block) % 16 == 0, "lion_ddpm_fetch_noise: dst / block must be 16-byte aligned");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddpm_fetch_noise, (unsigned)cdivz(n / 4, 256), 256, 0, (float4*)dst, (const float4*)block, step_ptr, n / 4);
  return check_launch(&c, "lion_ddpm_fetch_noise");
}
extern "C" int lion_ddpm_set_step(int* step_ptr, float* t_out, int B, int t_index, void* stream) {
  LION_REQUIRE(step_ptr && t_out && B > 0 && t_index >= 0, "lion_ddpm_set_step: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddpm_set_step, 1, 64, 0, step_ptr, t_out, B, t_index, 0);
  return check_launch(&c, "lion_ddpm_set_step");
}
extern "C" int lion_ddpm_next_step(int* step_ptr, float* t_out, int B, void* stream) {
  LION_REQUIRE(step_ptr && t_out && B > 0, "lion_ddpm_next_step: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddpm_set_step, 1, 64, 0, step_ptr, t_out, B, 0, 1);
  return check_launch(&c, "lion_ddpm_next_step");
}

extern "C" int lion_ddim_update(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                                const int* step_ptr, size_t n, float* hist, void* stream) {
  LION_REQUIRE(x && eps && x_out && tables && step_ptr && n > 0, "lion_ddim_update: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddim_update, (unsigned)cdivz(n, 256), 256, 0, x, eps, noise, x_out, (const float4*)tables, step_ptr, n, hist);
  return check_launch(&c, "lion_ddim_update");
}
extern "C" int lion_ddim_set_step(int* step_ptr, float* t_out, const float* tables, int B, int S, int index, void* stream) {
  LION_REQUIRE(step_ptr && t_out && tables && B > 0 && S > 0 && index >= 0 && index < S, "lion_ddim_set_step: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddim_set_step, 1, 64, 0, step_ptr, t_out, (const float4*)tables, B, S, index, 0);
  return check_launch(&c, "lion_ddim_set_step");
}
extern "C" int lion_ddim_next_step(int* step_ptr, float* t_out, const float* tables, int B, int S, void* stream) {
  LION_REQUIRE(step_ptr && t_out && tables && B > 0 && S > 0, "lion_ddim_next_step: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_ddim_set_step, 1, 64, 0, step_ptr, t_out, (const float4*)tables, B, S, 0, 1);
  return check_launch(&c, "lion_ddim_next_step");
}

extern "C" int lion_scheduler_step(const float* x, const float* eps, const float* noise, float* x_out, const float* tables,
                                   const int* step_ptr, size_t n, void* stream) {
  LION_REQUIRE(x && eps && x_out && tables && step_ptr && n > 0, "lion_scheduler_step: bad arguments");
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_sched_step, (unsigned)cdivz(n, 256), 256, 0, x, eps, noise ? noise : x, x_out, (const float4*)tables, step_ptr, n);
  return check_launch(&c, "lion_scheduler_step");
}

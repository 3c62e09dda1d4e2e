// lion_b200 -- the seven point<->voxel / neighbourhood operators of the reference's pvcnn
// extension, in the reference's own tensor layouts ([B,C,N] channel-major, flat voxel index
// x*r^2 + y*r + z), as stand-alone sm_90a kernels behind the C ABI (include/lion_b200.h).
//
// These are the drop-in for third_party/pvcnn/functional/src/bindings.cpp:10-37 (forward
// functions).  The fused network path (unet.cu) uses its own packed layouts and kernels; the
// index-producing device functions (FPS, ball query, 3-NN, voxel index) are shared through
// point_core.cuh so both paths give identical indices.
//
// Unlike the reference (grid = batch size, legacy default stream, exit(-1) on error) every
// kernel here is sized over B x work, launched on the caller's stream and reports errors by
// return code.
#include "common.cuh"
#include "point_core.cuh"
#include "../../include/lion_b200.h"

namespace lion {

// ------------------------------------------------------------------------------------
// avg_voxelize  (reference: voxelization/vox.cu:18-34, :48-72; vox.cpp:17-43)
// ------------------------------------------------------------------------------------
__global__ void k_grid_stats(const int* __restrict__ coords, int* __restrict__ ind, int* __restrict__ cnt,
                             int N, int r) {
  int b = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int* c = coords + (size_t)b * 3 * N;
  int v = c[i] * r * r + c[i + N] * r + c[i + 2 * N];
  ind[(size_t)b * N + i] = v;
  atomicAdd(cnt + (size_t)b * r * r * r + v, 1);
}

// one thread per (channel, point): coalesced feature reads, scattered atomics
__global__ void k_avg_voxelize(const float* __restrict__ feat, const int* __restrict__ ind,
                               const int* __restrict__ cnt, float* __restrict__ out, int C, int N, int r3) {
  int b = blockIdx.z;
  int c = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int pos = ind[(size_t)b * N + i];
  int k = cnt[(size_t)b * r3 + pos];
  if (k > 0) {
    float inv = 1.0f / (float)k;   // reference: 1.0 / static_cast<float>(cur_cnt), then float
    atomicAdd(out + ((size_t)b * C + c) * r3 + pos, feat[((size_t)b * C + c) * N + i] * inv);
  }
}

// ------------------------------------------------------------------------------------
// trilinear_devoxelize (reference: interpolate/trilinear_devox.cu:21-105)
// ------------------------------------------------------------------------------------
__global__ void k_trilinear_devox(const float* __restrict__ coords, const float* __restrict__ feat,
                                  int* __restrict__ inds, float* __restrict__ wgts, float* __restrict__ outs,
                                  int C, int N, int r, int is_training, int c_per_block) {
  int b = blockIdx.z;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* co = coords + (size_t)b * 3 * N;
  int idx[8];
  float w[8];
  trilinear_corners(co[i], co[i + N], co[i + 2 * N], r, idx, w);
  if (is_training && blockIdx.y == 0) {
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      wgts[((size_t)b * 8 + k) * N + i] = w[k];
      inds[((size_t)b * 8 + k) * N + i] = idx[k];
    }
  }
  int r3 = r * r * r;
  int c0 = blockIdx.y * c_per_block;
  int c1 = min(C, c0 + c_per_block);
  for (int c = c0; c < c1; ++c) {
    const float* f = feat + ((size_t)b * C + c) * r3;
    // same association as the reference: ((((w0 f0 + w1 f1) + w2 f2) + ...) + w7 f7)
    float acc = w[0] * __ldg(f + idx[0]);
#pragma unroll
    for (int k = 1; k < 8; ++k) acc = acc + w[k] * __ldg(f + idx[k]);
    outs[((size_t)b * C + c) * N + i] = acc;
  }
}

// ------------------------------------------------------------------------------------
// furthest point sampling (reference: sampling/sampling.cu:86-167) -- see point_core.cuh
// ------------------------------------------------------------------------------------
template <int A, int C, bool FULL>
__global__ void __launch_bounds__(FPS_THREADS)
k_fps_soa(const float* __restrict__ coords, int* __restrict__ idx_out, int N, int M, int VT) {
  extern __shared__ float s_fps[];
  int b = blockIdx.x;
  const float* c = coords + (size_t)b * 3 * N;
  int* io = idx_out + (size_t)b * M;
  fps_block_emit<A, C, FULL>([&](int k, float& x, float& y, float& z) { x = c[k]; y = c[k + N]; z = c[k + 2 * N]; },
                             [&](int j, int k, float, float, float) { io[j] = k; }, N, M, VT, s_fps);
}

__global__ void k_gather(const float* __restrict__ feat, const int* __restrict__ idx, float* __restrict__ out,
                         int C, int N, int M) {
  int b = blockIdx.z, c = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  out[((size_t)b * C + c) * M + j] = feat[((size_t)b * C + c) * N + idx[(size_t)b * M + j]];
}

// ------------------------------------------------------------------------------------
// ball query (reference: ball_query/ball_query.cu:19-50): one warp per centre
// ------------------------------------------------------------------------------------
__global__ void k_ball_query_soa(const float* __restrict__ centers, const float* __restrict__ points,
                                 int* __restrict__ out, int N, int M, float r2, int K) {
  int b = blockIdx.y;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warp >= M) return;
  const float* ce = centers + (size_t)b * 3 * M;
  const float* pt = points + (size_t)b * 3 * N;
  float cx = ce[warp], cy = ce[warp + M], cz = ce[warp + 2 * M];
  ball_query_warp([&](int k, float& x, float& y, float& z) { x = pt[k]; y = pt[k + N]; z = pt[k + 2 * N]; },
                  cx, cy, cz, r2, N, K, out + ((size_t)b * M + warp) * K);
}

__global__ void k_grouping(const float* __restrict__ feat, const int* __restrict__ idx, float* __restrict__ out,
                           int C, int N, int MU) {
  int b = blockIdx.z, c = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= MU) return;
  out[((size_t)b * C + c) * MU + j] = feat[((size_t)b * C + c) * N + idx[(size_t)b * MU + j]];
}

// ------------------------------------------------------------------------------------
// 3-NN + interpolation (reference: interpolate/neighbor_interpolate.cu:20-75, :90-116)
// ------------------------------------------------------------------------------------
__global__ void k_three_nn_soa(const float* __restrict__ points, const float* __restrict__ centers,
                               int* __restrict__ idx, float* __restrict__ wgt, int N, int M) {
  int b = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  extern __shared__ float s_c[];   // [3][tile]
  const float* pt = points + (size_t)b * 3 * N;
  const float* ce = centers + (size_t)b * 3 * M;
  float ux = 0, uy = 0, uz = 0;
  if (j < N) { ux = pt[j]; uy = pt[j + N]; uz = pt[j + 2 * N]; }
  ThreeNN st;
  st.init();
  const int TILE = 1024;
  for (int k0 = 0; k0 < M; k0 += TILE) {
    int n = min(TILE, M - k0);
    __syncthreads();
    for (int t = threadIdx.x; t < n; t += blockDim.x) {
      s_c[t] = ce[k0 + t]; s_c[TILE + t] = ce[k0 + t + M]; s_c[2 * TILE + t] = ce[k0 + t + 2 * M];
    }
    __syncthreads();
    for (int k = 0; k < n; ++k) st.push(sqdist_ref(ux - s_c[k], uy - s_c[TILE + k], uz - s_c[2 * TILE + k]), k0 + k);
  }
  if (j >= N) return;
  float w0, w1, w2;
  st.weights(w0, w1, w2);
  size_t o = (size_t)b * 3 * N + j;
  idx[o] = st.i0; idx[o + N] = st.i1; idx[o + 2 * N] = st.i2;
  wgt[o] = w0; wgt[o + N] = w1; wgt[o + 2 * N] = w2;
}

__global__ void k_three_interp(const float* __restrict__ cf, const int* __restrict__ idx,
                               const float* __restrict__ wgt, float* __restrict__ out, int C, int N, int M) {
  int b = blockIdx.z, c = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  size_t o = (size_t)b * 3 * N + j;
  const float* f = cf + ((size_t)b * C + c) * M;
  out[((size_t)b * C + c) * N + j] = f[idx[o]] * wgt[o] + f[idx[o + N]] * wgt[o + N] + f[idx[o + 2 * N]] * wgt[o + 2 * N];
}

// ------------------------------------------------------------------------------------
// Voxelization.forward's coordinate part (reference: models/pvcnn2_ada.py:173-188)
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(VOX_THREADS)
k_voxel_coords_soa(const float* __restrict__ coords, float* __restrict__ norm_coords, int* __restrict__ vox,
                   int N, int r, int normalize, float eps) {
  int b = blockIdx.x;
  const float* c = coords + (size_t)b * 3 * N;
  __shared__ float s_stat[4];
  vox_stats_block<VOX_THREADS / 32>([&](int k, float& x, float& y, float& z) { x = c[k]; y = c[k + N]; z = c[k + 2 * N]; }, N,
                                    3 * (int)gridDim.x, 3LL * b, s_stat);
  float mx = s_stat[0], my = s_stat[1], mz = s_stat[2], nrm = s_stat[3];
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    float v[3];
    vox_normalize(c[k] - mx, c[k + N] - my, c[k + 2 * N] - mz, nrm, r, normalize, eps, v);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      norm_coords[((size_t)b * 3 + a) * N + k] = v[a];
      vox[((size_t)b * 3 + a) * N + k] = (int)rintf(v[a]);
    }
  }
}

// ------------------------------------------------------------------------------------
// backward kernels of the five differentiable operators (SURVEY.md 8f rank 4; reference: voxelization/vox.cu:86-110,
// interpolate/trilinear_devox.cu:119-162, grouping/grouping.cu:58-77, interpolate/neighbor_interpolate.cu:145-170,
// sampling/sampling.cu:52-66).  The reference launches one CTA per shape and loops over channels inside a thread;
// here the grid covers (rows, channel, shape) so all SMs take part and every access along rows is coalesced.
// Scatter-type gradients accumulate with fp32 atomics like the reference (order-dependent in the last bits).
// ------------------------------------------------------------------------------------
// avg_voxelize backward is a pure gather: grad_x[b][c][i] = grad_y[b][c][ind[i]] * (1 / cnt[ind[i]])
__global__ void k_avg_voxelize_bwd(const float* __restrict__ gy, const int* __restrict__ ind, const int* __restrict__ cnt,
                                   float* __restrict__ gx, int C, int N, int r3) {
  int b = blockIdx.z, c = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  int pos = ind[(size_t)b * N + i];
  int n = cnt[(size_t)b * r3 + pos];
  float g = 0.0f;
  if (n > 0) g = gy[((size_t)b * C + c) * r3 + pos] * (float)(1.0 / (double)(float)n);   // vox.cu:101-104
  gx[((size_t)b * C + c) * N + i] = g;
}
// trilinear devoxelize backward: 8 weighted scatter-adds per (point, channel) into the (pre-zeroed) grid gradient
__global__ void k_trilinear_devox_bwd(const float* __restrict__ gy, const int* __restrict__ inds, const float* __restrict__ wgts,
                                      float* __restrict__ gx, int C, int N, int r3) {
  int b = blockIdx.z, c = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  float g = gy[((size_t)b * C + c) * N + i];
  const int* id = inds + (size_t)b * 8 * N + i;
  const float* w = wgts + (size_t)b * 8 * N + i;
  float* dst = gx + ((size_t)b * C + c) * r3;
#pragma unroll
  for (int k = 0; k < 8; ++k) atomicAdd(dst + id[(size_t)k * N], w[(size_t)k * N] * g);
}
// grouping backward: grad_x[b][c][idx[b][j][k]] += grad_y[b][c][j][k]
__global__ void k_grouping_bwd(const float* __restrict__ gy, const int* __restrict__ idx, float* __restrict__ gx, int C, int N, int MU) {
  int b = blockIdx.z, c = blockIdx.y;
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= MU) return;
  atomicAdd(gx + ((size_t)b * C + c) * N + idx[(size_t)b * MU + i], gy[((size_t)b * C + c) * MU + i]);
}
// 3-NN interpolation backward: grad_cf[b][c][idx_k[j]] += grad_y[b][c][j] * w_k[j], k = 0..2
__global__ void k_three_interp_bwd(const float* __restrict__ gy, const int* __restrict__ idx, const float* __restrict__ wgt,
                                   float* __restrict__ gx, int C, int N, int M) {
  int b = blockIdx.z, c = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= N) return;
  float g = gy[((size_t)b * C + c) * N + j];
  size_t o = (size_t)b * 3 * N + j;
  float* dst = gx + ((size_t)b * C + c) * M;
  atomicAdd(dst + idx[o], g * wgt[o]);
  atomicAdd(dst + idx[o + N], g * wgt[o + N]);
  atomicAdd(dst + idx[o + 2 * (size_t)N], g * wgt[o + 2 * (size_t)N]);
}
// gather backward: grad_x[b][c][idx[b][j]] += grad_y[b][c][j]
__global__ void k_gather_bwd(const float* __restrict__ gy, const int* __restrict__ idx, float* __restrict__ gx, int C, int N, int M) {
  int b = blockIdx.z, c = blockIdx.y;
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  atomicAdd(gx + ((size_t)b * C + c) * N + idx[(size_t)b * M + j], gy[((size_t)b * C + c) * M + j]);
}

}  // namespace lion

// =====================================================================================
// C ABI
// =====================================================================================
using namespace lion;

static inline Ctx tmp_ctx(void* stream) {
  Ctx c;
  c.stream = (cudaStream_t)stream;
  return c;
}

extern "C" int lion_avg_voxelize(const float* feat, const int* coords, float* out, int* ind, int* cnt,
                                 int B, int C, int N, int r, void* stream) {
  LION_REQUIRE(feat && coords && out && ind && cnt, "lion_avg_voxelize: null pointer");
  LION_REQUIRE(B > 0 && C > 0 && N > 0 && r > 0 && r <= 256, "lion_avg_voxelize: bad sizes B=%d C=%d N=%d r=%d", B, C, N, r);
  Ctx c = tmp_ctx(stream);
  size_t r3 = (size_t)r * r * r;
  // outputs are accumulated into: zero them here (the reference's wrapper allocates zeros, vox.cpp:33-38)
  LION_TRY(memset_async(&c, out, 0, sizeof(float) * B * C * r3));
  LION_TRY(memset_async(&c, cnt, 0, sizeof(int) * B * r3));
  LION_LAUNCH(&c, k_grid_stats, dim3(cdiv(N, 256), B), 256, 0, coords, ind, cnt, N, r);
  LION_LAUNCH(&c, k_avg_voxelize, dim3(cdiv(N, 256), C, B), 256, 0, feat, ind, cnt, out, C, N, (int)r3);
  return check_launch(&c, "lion_avg_voxelize");
}

extern "C" int lion_trilinear_devoxelize(const float* grid, const float* coords, float* out, int* inds, float* wgts,
                                         int B, int C, int N, int r, int is_training, void* stream) {
  LION_REQUIRE(grid && coords && out, "lion_trilinear_devoxelize: null pointer");
  LION_REQUIRE(!is_training || (inds && wgts), "lion_trilinear_devoxelize: is_training needs inds/wgts");
  LION_REQUIRE(B > 0 && C > 0 && N > 0 && r > 0, "lion_trilinear_devoxelize: bad sizes");
  Ctx c = tmp_ctx(stream);
  int cpb = 8;
  LION_LAUNCH(&c, k_trilinear_devox, dim3(cdiv(N, 128), cdiv(C, cpb), B), 128, 0, coords, grid, inds, wgts, out,
              C, N, r, is_training, cpb);
  return check_launch(&c, "lion_trilinear_devoxelize");
}

extern "C" int lion_furthest_point_sampling(const float* coords, int* idx, int B, int N, int M, void* stream) {
  LION_REQUIRE(coords && idx, "lion_furthest_point_sampling: null pointer");
  LION_REQUIRE(B > 0 && N > 0 && M > 0, "lion_furthest_point_sampling: bad sizes");
  LION_REQUIRE(N <= FPS_MAX_N, "lion_furthest_point_sampling: N=%d exceeds %d", N, FPS_MAX_N);
  Ctx c = tmp_ctx(stream);
  const int VT = fps_virtual_threads(N);
#define LION_FPS_CALL(A_, C_, F_)                                                                                          \
  do {                                                                                                                     \
    if (fps_smem_bytes(N) > 48 * 1024)                                                                                     \
      LION_CHECK_CUDA(cudaFuncSetAttribute(k_fps_soa<A_, C_, F_>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); \
    LION_LAUNCH(&c, (k_fps_soa<A_, C_, F_>), B, FPS_THREADS, fps_smem_bytes(N), coords, idx, N, M, VT);                    \
  } while (0)
  LION_FPS_DISPATCH(N, VT, LION_FPS_CALL);
#undef LION_FPS_CALL
  return check_launch(&c, "lion_furthest_point_sampling");
}

extern "C" int lion_gather(const float* feat, const int* idx, float* out, int B, int C, int N, int M, void* stream) {
  LION_REQUIRE(feat && idx && out, "lion_gather: null pointer");
  LION_REQUIRE(B > 0 && C > 0 && N > 0 && M > 0, "lion_gather: bad sizes");
  Ctx c = tmp_ctx(stream);
  LION_LAUNCH(&c, k_gather, dim3(cdiv(M, 128), C, B), 128, 0, feat, idx, out, C, N, M);
  return check_launch(&c, "lion_gather");
}

extern "C" int lion_ball_query(const float* centers, const float* points, int* out, int B, int N, int M,
                               float radius, int K, void* stream) {
  LION_REQUIRE(centers && points && out, "lion_ball_query: null pointer");
  LION_REQUIRE(B > 0 && N > 0 && M > 0 && K > 0 && K <= 32, "lion_ball_query: bad sizes (K<=32)");
  Ctx c = tmp_ctx(stream);
  float r2 = radius * radius;   // float product, as ball_query.cpp passes radius*radius computed in float
  LION_LAUNCH(&c, k_ball_query_soa, dim3(cdiv(M * 32, 256), B), 256, 0, centers, points, out, N, M, r2, K);
  return check_launch(&c, "lion_ball_query");
}

extern "C" int lion_grouping(const float* feat, const int* idx, float* out, int B, int C, int N, int M, int U,
                             void* stream) {
  LION_REQUIRE(feat && idx && out, "lion_grouping: null pointer");
  LION_REQUIRE(B > 0 && C > 0 && N > 0 && M > 0 && U > 0, "lion_grouping: bad sizes");
  Ctx c = tmp_ctx(stream);
  LION_LAUNCH(&c, k_grouping, dim3(cdiv(M * U, 256), C, B), 256, 0, feat, idx, out, C, N, M * U);
  return check_launch(&c, "lion_grouping");
}

extern "C" int lion_three_nn_interpolate(const float* points, const float* centers, const float* cfeat, float* out,
                                         int* idx, float* wgt, int B, int C, int N, int M, void* stream) {
  LION_REQUIRE(points && centers && cfeat && out && idx && wgt, "lion_three_nn_interpolate: null pointer");
  LION_REQUIRE(B > 0 && C > 0 && N > 0 && M > 0, "lion_three_nn_interpolate: bad sizes");
  Ctx c = tmp_ctx(stream);
  LION_LAUNCH(&c, k_three_nn_soa, dim3(cdiv(N, 128), B), 128, 3 * 1024 * sizeof(float), points, centers, idx, wgt, N, M);
  LION_LAUNCH(&c, k_three_interp, dim3(cdiv(N, 128), C, B), 128, 0, cfeat, idx, wgt, out, C, N, M);
  return check_launch(&c, "lion_three_nn_interpolate");
}

extern "C" int lion_voxel_coords(const float* coords, float* norm_coords, int* vox, int B, int N, int r,
                                 int normalize, float eps, void* stream) {
  LION_REQUIRE(coords && norm_coords && vox, "lion_voxel_coords: null pointer");
  LION_REQUIRE(B > 0 && N > 0 && r > 0, "lion_voxel_coords: bad sizes");
  Ctx c = tmp_ctx(stream);
  LION_LAUNCH(&c, k_voxel_coords_soa, B, VOX_THREADS, 0, coords, norm_coords, vox, N, r, normalize, eps);
  return check_launch(&c, "lion_voxel_coords");
}

// ---- backward entry points (reference: src/bindings.cpp:12-13,19-20,24-25,29-30,33-34) ------------------------------
extern "C" int lion_avg_voxelize_backward(const float* grad_y, const int* ind, const int* cnt, float* grad_x, int B, int C,
                                          int N, int r, void* stream) {
  LION_REQUIRE(grad_y && ind && cnt && grad_x && B > 0 && C > 0 && N > 0 && r > 0, "lion_avg_voxelize_backward: bad arguments");
  Ctx c = tmp_ctx(stream);
  LION_LAUNCH(&c, k_avg_voxelize_bwd, dim3(cdiv(N, 256), C, B), 256, 0, grad_y, ind, cnt, grad_x, C, N, r * r * r);
  return check_launch(&c, "lion_avg_voxelize_backward");
}
extern "C" int lion_trilinear_devoxelize_backward(const float* grad_y, const int* inds, const float* wgts, float* grad_x, int B,
                                                  int C, int N, int r, void* stream) {
  LION_REQUIRE(grad_y && inds && wgts && grad_x && B > 0 && C > 0 && N > 0 && r > 0, "lion_trilinear_devoxelize_backward: bad arguments");
  Ctx c = tmp_ctx(stream);
  const int r3 = r * r * r;
  LION_TRY(memset_async(&c, grad_x, 0, sizeof(float) * (size_t)B * C * r3));
  LION_LAUNCH(&c, k_trilinear_devox_bwd, dim3(cdiv(N, 256), C, B), 256, 0, grad_y, inds, wgts, grad_x, C, N, r3);
  return check_launch(&c, "lion_trilinear_devoxelize_backward");
}
extern "C" int lion_grouping_backward(const float* grad_y, const int* idx, float* grad_x, int B, int C, int N, int M, int U,
                                      void* stream) {
  LION_REQUIRE(grad_y && idx && grad_x && B > 0 && C > 0 && N > 0 && M > 0 && U > 0, "lion_grouping_backward: bad arguments");
  Ctx c = tmp_ctx(stream);
  LION_TRY(memset_async(&c, grad_x, 0, sizeof(float) * (size_t)B * C * N));
  LION_LAUNCH(&c, k_grouping_bwd, dim3(cdiv(M * U, 256), C, B), 256, 0, grad_y, idx, grad_x, C, N, M * U);
  return check_launch(&c, "lion_grouping_backward");
}
extern "C" int lion_three_nn_interpolate_backward(const float* grad_y, const int* idx, const float* wgt, float* grad_x, int B,
                                                  int C, int N, int M, void* stream) {
  LION_REQUIRE(grad_y && idx && wgt && grad_x && B > 0 && C > 0 && N > 0 && M > 0, "lion_three_nn_interpolate_backward: bad arguments");
  Ctx c = tmp_ctx(stream);
  LION_TRY(memset_async(&c, grad_x, 0, sizeof(float) * (size_t)B * C * M));
  LION_LAUNCH(&c, k_three_interp_bwd, dim3(cdiv(N, 256), C, B), 256, 0, grad_y, idx, wgt, grad_x, C, N, M);
  return check_launch(&c, "lion_three_nn_interpolate_backward");
}
extern "C" int lion_gather_backward(const float* grad_y, const int* idx, float* grad_x, int B, int C, int N, int M, void* stream) {
  LION_REQUIRE(grad_y && idx && grad_x && B > 0 && C > 0 && N > 0 && M > 0, "lion_gather_backward: bad arguments");
  Ctx c = tmp_ctx(stream);
  LION_TRY(memset_async(&c, grad_x, 0, sizeof(float) * (size_t)B * C * N));
  LION_LAUNCH(&c, k_gather_bwd, dim3(cdiv(M, 256), C, B), 256, 0, grad_y, idx, grad_x, C, N, M);
  return check_launch(&c, "lion_gather_backward");
}

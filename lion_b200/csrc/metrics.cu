// lion_b200 -- Chamfer nearest-neighbour kernels for the generation metrics that follow sampling
// (SURVEY.md 8f rank 2).
//
// Reference: third_party/ChamferDistancePytorch/chamfer3D/chamfer3D.cu:12-143 (NmDistanceKernel,
// launched twice as <<<dim3(32,16,1),512>>> by chamfer_cuda_forward) and its use in
// utils/evaluation_metrics_fast.py:272-340 (_pairwise_EMD_CD_: one sample cloud expanded against a
// batch of reference clouds, dl.mean(1) + dr.mean(1)).
//
// Semantics kept bit for bit:
//   * d = (x2-x1)^2 + (y2-y1)^2 + (z2-z1)^2 with the contraction nvcc applies to the reference
//     source (t = dy*dy; t = fma(dx,dx,t); t = fma(dz,dz,t) -- read off the reference's SASS, the
//     same pattern as the pvcnn kernels, common.cuh: sqdist_ref);
//   * the first candidate is always taken, later ones only when strictly smaller, also across the
//     reference's 512-point chunks (`result > best`): the lowest index wins exact ties.
// Design: the candidate cloud is staged once in shared memory as SoA (three broadcast LDS per
// candidate), every thread keeps Q query points and their running (best, index) in registers, so
// a candidate costs 3 LDS + Q x 8 FP32/select instructions; the pairwise kernel handles both
// directions of one (sample, reference) pair per CTA and reduces the two means in a fixed order
// (deterministic, no atomics, no [Nr, N, 3] expansion of the sample cloud).
#include "common.cuh"
#include "../../include/lion_b200.h"

namespace lion {

constexpr int CD_THREADS = 128;
constexpr int CD_Q = 4;            // query points per thread
constexpr int CD_CHUNK = 2048;     // candidates staged per pass (24 KB)

// one direction: queries q[b][n][3] against candidates c[b][m][3] -> dist[b][n], idx[b][n]
__global__ void __launch_bounds__(CD_THREADS)
k_chamfer_nn(const float* __restrict__ q, const float* __restrict__ c, float* __restrict__ dist, int* __restrict__ idx,
             int n, int m) {
  __shared__ float sx[CD_CHUNK], sy[CD_CHUNK], sz[CD_CHUNK];
  const int b = blockIdx.y;
  const float* qb = q + (size_t)b * n * 3;
  const float* cb = c + (size_t)b * m * 3;
  float x1[CD_Q], y1[CD_Q], z1[CD_Q], best[CD_Q];
  int bi[CD_Q];
#pragma unroll
  for (int u = 0; u < CD_Q; ++u) {
    int j = (blockIdx.x * CD_Q + u) * CD_THREADS + threadIdx.x;
    int jj = j < n ? j : 0;
    x1[u] = qb[jj * 3 + 0]; y1[u] = qb[jj * 3 + 1]; z1[u] = qb[jj * 3 + 2];
    best[u] = 0.0f; bi[u] = 0;
  }
  for (int k0 = 0; k0 < m; k0 += CD_CHUNK) {
    const int kn = min(CD_CHUNK, m - k0);
    __syncthreads();
    for (int k = threadIdx.x; k < kn; k += CD_THREADS) {
      sx[k] = cb[(size_t)(k0 + k) * 3 + 0]; sy[k] = cb[(size_t)(k0 + k) * 3 + 1]; sz[k] = cb[(size_t)(k0 + k) * 3 + 2];
    }
    __syncthreads();
    int k = 0;
    if (k0 == 0) {            // the first candidate is taken unconditionally (reference: `k==0 || d<best`)
#pragma unroll
      for (int u = 0; u < CD_Q; ++u) { best[u] = sqdist_ref(sx[0] - x1[u], sy[0] - y1[u], sz[0] - z1[u]); bi[u] = 0; }
      k = 1;
    }
#pragma unroll 4
    for (; k < kn; ++k) {
      const float cx = sx[k], cy = sy[k], cz = sz[k];
#pragma unroll
      for (int u = 0; u < CD_Q; ++u) {
        float d = sqdist_ref(cx - x1[u], cy - y1[u], cz - z1[u]);
        if (d < best[u]) { best[u] = d; bi[u] = k0 + k; }
      }
    }
  }
#pragma unroll
  for (int u = 0; u < CD_Q; ++u) {
    int j = (blockIdx.x * CD_Q + u) * CD_THREADS + threadIdx.x;
    if (j < n) { dist[(size_t)b * n + j] = best[u]; if (idx) idx[(size_t)b * n + j] = bi[u]; }
  }
}

// pairwise Chamfer matrix: out[i][j] = mean_n min_m d(s_i[n], r_j[m]) + mean_m min_n d(r_j[m], s_i[n])
// one CTA per (i, j); both clouds live in shared memory (n, m <= CD_PW_MAX points each)
constexpr int CD_PW_MAX = 2048;
constexpr int CD_PW_THREADS = 256;

__device__ __forceinline__ float cd_direction_sum(const float* qx, const float* qy, const float* qz, int n,
                                                  const float* cx, const float* cy, const float* cz, int m) {
  // every thread owns queries t, t + T, ... (<= CD_PW_MAX / T = 8) and scans all candidates
  constexpr int QP = CD_PW_MAX / CD_PW_THREADS;
  float x1[QP], y1[QP], z1[QP], best[QP];
#pragma unroll
  for (int u = 0; u < QP; ++u) {
    int j = u * CD_PW_THREADS + threadIdx.x;
    int jj = j < n ? j : 0;
    x1[u] = qx[jj]; y1[u] = qy[jj]; z1[u] = qz[jj];
    best[u] = sqdist_ref(cx[0] - x1[u], cy[0] - y1[u], cz[0] - z1[u]);
  }
#pragma unroll 2
  for (int k = 1; k < m; ++k) {
    const float ax = cx[k], ay = cy[k], az = cz[k];
#pragma unroll
    for (int u = 0; u < QP; ++u) {
      float d = sqdist_ref(ax - x1[u], ay - y1[u], az - z1[u]);
      best[u] = d < best[u] ? d : best[u];
    }
  }
  float s = 0.0f;
#pragma unroll
  for (int u = 0; u < QP; ++u) s += (u * CD_PW_THREADS + threadIdx.x < n) ? best[u] : 0.0f;
  return s;
}

__global__ void __launch_bounds__(CD_PW_THREADS)
k_chamfer_pairwise(const float* __restrict__ samples, const float* __restrict__ refs, float* __restrict__ out,
                   int n, int m, int n_ref) {
  extern __shared__ float sm[];     // s: x,y,z [n] ; r: x,y,z [m] ; reduction scratch
  float* sxp = sm; float* syp = sxp + CD_PW_MAX; float* szp = syp + CD_PW_MAX;
  float* rxp = szp + CD_PW_MAX; float* ryp = rxp + CD_PW_MAX; float* rzp = ryp + CD_PW_MAX;
  float* red = rzp + CD_PW_MAX;     // [2][warps]
  const int i = blockIdx.y, j = blockIdx.x;
  const float* s = samples + (size_t)i * n * 3;
  const float* r = refs + (size_t)j * m * 3;
  for (int k = threadIdx.x; k < n; k += CD_PW_THREADS) { sxp[k] = s[k * 3]; syp[k] = s[k * 3 + 1]; szp[k] = s[k * 3 + 2]; }
  for (int k = threadIdx.x; k < m; k += CD_PW_THREADS) { rxp[k] = r[k * 3]; ryp[k] = r[k * 3 + 1]; rzp[k] = r[k * 3 + 2]; }
  __syncthreads();
  float a = cd_direction_sum(sxp, syp, szp, n, rxp, ryp, rzp, m);     // sample -> reference ("dl")
  float c = cd_direction_sum(rxp, ryp, rzp, m, sxp, syp, szp, n);     // reference -> sample ("dr")
  a = warp_sum(a); c = warp_sum(c);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { red[warp] = a; red[CD_PW_THREADS / 32 + warp] = c; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float ta = 0.0f, tc = 0.0f;
    for (int w = 0; w < CD_PW_THREADS / 32; ++w) { ta += red[w]; tc += red[CD_PW_THREADS / 32 + w]; }
    out[(size_t)i * n_ref + j] = ta / (float)n + tc / (float)m;
  }
}

}  // namespace lion

using namespace lion;

extern "C" int lion_chamfer_forward(const float* xyz1, const float* xyz2, float* dist1, float* dist2, int* idx1, int* idx2,
                                    int B, int N, int M, void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && dist1 && dist2 && B > 0 && N > 0 && M > 0, "lion_chamfer_forward: bad arguments");
  LION_REQUIRE(B <= 65535, "lion_chamfer_forward: at most 65535 cloud pairs per call (got %d)", B);
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_chamfer_nn, dim3(cdiv(N, CD_THREADS * CD_Q), B), CD_THREADS, 0, xyz1, xyz2, dist1, idx1, N, M);
  LION_LAUNCH(&c, k_chamfer_nn, dim3(cdiv(M, CD_THREADS * CD_Q), B), CD_THREADS, 0, xyz2, xyz1, dist2, idx2, M, N);
  return check_launch(&c, "lion_chamfer_forward");
}

extern "C" int lion_chamfer_pairwise(const float* samples, const float* refs, float* out, int n_sample, int n_ref, int N, int M,
                                     void* stream) {
  LION_REQUIRE(samples && refs && out && n_sample > 0 && n_ref > 0 && N > 0 && M > 0, "lion_chamfer_pairwise: bad arguments");
  LION_REQUIRE(N <= CD_PW_MAX && M <= CD_PW_MAX, "lion_chamfer_pairwise: clouds of at most %d points (got %d, %d)", CD_PW_MAX, N, M);
  LION_REQUIRE(n_sample <= 65535, "lion_chamfer_pairwise: at most 65535 sample clouds per call (got %d)", n_sample);
  Ctx c;
  c.stream = (cudaStream_t)stream;
  const size_t smem = (6 * CD_PW_MAX + 2 * (CD_PW_THREADS / 32)) * sizeof(float);
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_chamfer_pairwise, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}
  LION_LAUNCH(&c, k_chamfer_pairwise, dim3(n_ref, n_sample), CD_PW_THREADS, smem, samples, refs, out, N, M, n_ref);
  return check_launch(&c, "lion_chamfer_pairwise");
}

// =====================================================================================
// approximate earth mover's distance (SURVEY.md 8f rank 2, second half)
//
// Reference: third_party/PyTorchEMD/cuda/emd_kernel.cu:23-170 (approxmatch<<<32,512>>>: ten
// annealing levels -4^7 .. -4^-1, 0 of a soft assignment with row / column capacities, writing a
// dense match[b][m][n]) followed by :196-246 (matchcost<<<32,512>>>: sum of d^2 * match), as called by
// third_party/PyTorchEMD/emd_nograd.py:9-45 and utils/evaluation_metrics_fast.py:122-147 (emd_approx).
//
// Here: ONE kernel, one CTA per cloud pair; both clouds and the four capacity / ratio vectors live
// in shared memory, every thread owns EMD_Q rows (points of xyz1) whose coordinates stay in registers,
// and the cost sum(d^2 * w) is accumulated where the reference adds w into `match`, so the
// [b][m][n] matrix (16 MB per pair at 2048 points) is never written.  Arithmetic follows the
// reference expression by expression (same __expf, same per-thread summation order over the
// other cloud) so the annealing iterates agree to rounding; only the final cost is summed in a
// different order (per level instead of per matrix element).
// =====================================================================================
namespace lion {

constexpr int EMD_THREADS = 512;
constexpr int EMD_Q = 4;                      // rows per thread -> n, m <= 2048
constexpr int EMD_MAX = EMD_THREADS * EMD_Q;

__device__ __forceinline__ float emd_d2(float x1, float y1, float z1, float x2, float y2, float z2) {
  return (x2 - x1) * (x2 - x1) + (y2 - y1) * (y2 - y1) + (z2 - z1) * (z2 - z1);
}

// pair p: xyz1 = a[(p / nb) or p], xyz2 = b[(p % nb) or p]
__global__ void __launch_bounds__(EMD_THREADS)
k_emd_approx(const float* __restrict__ a, const float* __restrict__ bb, float* __restrict__ out, int n, int m, int nb, int pairwise) {
  extern __shared__ float sm[];
  float4* p1 = reinterpret_cast<float4*>(sm);            // [n] x,y,z of xyz1 + ratioL
  float4* p2 = p1 + EMD_MAX;                             // [m] x,y,z of xyz2 + (remainR | ratioR)
  float* remainL = reinterpret_cast<float*>(p2 + EMD_MAX);
  float* remainR = remainL + EMD_MAX;
  float* ratioR = remainR + EMD_MAX;
  float* red = ratioR + EMD_MAX;                          // [EMD_THREADS]
  const int p = blockIdx.x, tid = threadIdx.x;
  const float* xyz1 = a + (size_t)(pairwise ? p / nb : p) * n * 3;
  const float* xyz2 = bb + (size_t)(pairwise ? p % nb : p) * m * 3;
  float multiL, multiR;
  if (n >= m) { multiL = 1; multiR = n / m; } else { multiL = m / n; multiR = 1; }       // integer division as in the reference
  for (int k = tid; k < n; k += EMD_THREADS) { p1[k] = make_float4(xyz1[k * 3], xyz1[k * 3 + 1], xyz1[k * 3 + 2], 0.f); remainL[k] = multiL; }
  for (int l = tid; l < m; l += EMD_THREADS) { p2[l] = make_float4(xyz2[l * 3], xyz2[l * 3 + 1], xyz2[l * 3 + 2], 0.f); remainR[l] = multiR; }
  float cost = 0.0f;
  __syncthreads();
  for (int j = 7; j >= -2; j--) {
    float level = -powf(4.0f, j);
    if (j == -2) level = 0;
    // ---- pass 1: ratioL[k] = remainL[k] / (1e-9 + sum_l exp(level d) remainR[l]) ---------------
    for (int l = tid; l < m; l += EMD_THREADS) p2[l].w = remainR[l];
    __syncthreads();
    {
      float x1[EMD_Q], y1[EMD_Q], z1[EMD_Q], suml[EMD_Q];
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int k = u * EMD_THREADS + tid;
        float4 q = k < n ? p1[k] : make_float4(0.f, 0.f, 0.f, 0.f);
        x1[u] = q.x; y1[u] = q.y; z1[u] = q.z; suml[u] = 1e-9f;
      }
      for (int l = 0; l < m; ++l) {
        const float4 c = p2[l];
#pragma unroll
        for (int u = 0; u < EMD_Q; ++u) {
          float d = level * emd_d2(x1[u], y1[u], z1[u], c.x, c.y, c.z);
          float w = __expf(d) * c.w;
          suml[u] += w;
        }
      }
      __syncthreads();                                   // everyone is done reading p2[].w / p1[].w
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int k = u * EMD_THREADS + tid;
        if (k < n) p1[k].w = remainL[k] / suml[u];       // ratioL
      }
    }
    __syncthreads();
    // ---- pass 2: per column l: sumr, consumption -> ratioR[l], remainR[l] ----------------------
    {
      float x2[EMD_Q], y2[EMD_Q], z2[EMD_Q], sumr[EMD_Q];
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int l = u * EMD_THREADS + tid;
        float4 q = l < m ? p2[l] : make_float4(0.f, 0.f, 0.f, 0.f);
        x2[u] = q.x; y2[u] = q.y; z2[u] = q.z; sumr[u] = 0.0f;
      }
      for (int k = 0; k < n; ++k) {
        const float4 c = p1[k];
#pragma unroll
        for (int u = 0; u < EMD_Q; ++u) {
          float w = __expf(level * emd_d2(c.x, c.y, c.z, x2[u], y2[u], z2[u])) * c.w;
          sumr[u] += w;
        }
      }
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int l = u * EMD_THREADS + tid;
        if (l < m) {
          float r = remainR[l];
          float s = sumr[u] * r;
          float consumption = fminf(r / (s + 1e-9f), 1.0f);
          ratioR[l] = consumption * r;
          remainR[l] = fmaxf(0.0f, r - s);
        }
      }
    }
    __syncthreads();
    // ---- pass 3: w = exp(level d) ratioL[k] ratioR[l]  (the reference adds it to match[l][k]);
    //      cost += d2 * w;  remainL[k] = max(0, remainL[k] - sum_l w) -------------------------------
    for (int l = tid; l < m; l += EMD_THREADS) p2[l].w = ratioR[l];
    __syncthreads();
    {
      float x1[EMD_Q], y1[EMD_Q], z1[EMD_Q], rl[EMD_Q], suml[EMD_Q];
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int k = u * EMD_THREADS + tid;
        float4 q = k < n ? p1[k] : make_float4(0.f, 0.f, 0.f, 0.f);
        x1[u] = q.x; y1[u] = q.y; z1[u] = q.z; rl[u] = q.w; suml[u] = 0.0f;
      }
      for (int l = 0; l < m; ++l) {
        const float4 c = p2[l];
#pragma unroll
        for (int u = 0; u < EMD_Q; ++u) {
          float d2 = emd_d2(x1[u], y1[u], z1[u], c.x, c.y, c.z);
          float w = __expf(level * d2) * rl[u] * c.w;
          suml[u] += w;
          cost = fmaf(d2, w, cost);                      // rows k >= n carry rl = 0 -> w = 0
        }
      }
#pragma unroll
      for (int u = 0; u < EMD_Q; ++u) {
        int k = u * EMD_THREADS + tid;
        if (k < n) remainL[k] = fmaxf(0.0f, remainL[k] - suml[u]);
      }
    }
    __syncthreads();
  }
  // block sum in a fixed order
  cost = warp_sum(cost);
  if ((tid & 31) == 0) red[tid >> 5] = cost;
  __syncthreads();
  if (tid == 0) {
    float t = 0.0f;
    for (int w = 0; w < EMD_THREADS / 32; ++w) t += red[w];
    out[p] = t;
  }
}

}  // namespace lion

static int emd_launch(const float* a, const float* b, float* out, int pairs, int n, int m, int nb, int pairwise, void* stream) {
  Ctx c;
  c.stream = (cudaStream_t)stream;
  const size_t smem = (size_t)EMD_MAX * (2 * sizeof(float4) + 3 * sizeof(float)) + EMD_THREADS * sizeof(float);
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_emd_approx, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}
  LION_LAUNCH(&c, k_emd_approx, pairs, EMD_THREADS, smem, a, b, out, n, m, nb, pairwise);
  return check_launch(&c, "lion_emd_approx");
}

extern "C" int lion_emd_approx(const float* xyz1, const float* xyz2, float* cost, int B, int N, int M, void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && cost && B > 0 && N > 0 && M > 0, "lion_emd_approx: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_approx: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  return emd_launch(xyz1, xyz2, cost, B, N, M, 1, 0, stream);
}

extern "C" int lion_emd_pairwise(const float* samples, const float* refs, float* out, int n_sample, int n_ref, int N, int M,
                                 void* stream) {
  LION_REQUIRE(samples && refs && out && n_sample > 0 && n_ref > 0 && N > 0 && M > 0, "lion_emd_pairwise: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_pairwise: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  LION_REQUIRE((long long)n_sample * n_ref < (1LL << 31), "lion_emd_pairwise: too many pairs");
  return emd_launch(samples, refs, out, n_sample * n_ref, N, M, n_ref, 1, stream);
}

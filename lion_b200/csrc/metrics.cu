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
#include <climits>
#include <math_constants.h>
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

constexpr int EMD_LEVELS = 10;                // annealing levels -4^7 .. -4^-1, 0

// pair p: xyz1 = a[(p / nb) or p], xyz2 = b[(p % nb) or p]
// SAVE: also write level t's ratioL to ratios[p][t][0..n) and its ratioR to ratios[p][t][n..n+m) -- all that
// k_emd_backward needs to rebuild match[l][k] = sum_t exp(level_t d2(k,l)) ratioL_t[k] ratioR_t[l].
template <bool SAVE>
__global__ void __launch_bounds__(EMD_THREADS)
k_emd_approx(const float* __restrict__ a, const float* __restrict__ bb, float* __restrict__ out, float* __restrict__ ratios,
             int n, int m, int nb, int pairwise) {
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
    float* saved = SAVE ? ratios + ((size_t)p * EMD_LEVELS + (7 - j)) * (n + m) : nullptr;
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
        if (k < n) {
          p1[k].w = remainL[k] / suml[u];                // ratioL
          if (SAVE) saved[k] = p1[k].w;
        }
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
          if (SAVE) saved[n + l] = consumption * r;
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

// ---- backward (reference: emd_kernel.cu:280-353, matchcostgrad1 / matchcostgrad2) ---------------------------
//   grad1[k] = gc * sum_l 2 match[l][k] (xyz1_k - xyz2_l),   grad2[l] = gc * sum_k 2 match[l][k] (xyz2_l - xyz1_k)
// with match treated as a constant (the annealing is not differentiated), as in the reference.  match is rebuilt on
// the fly from the ratios k_emd_approx<true> saved, with the forward's d2 and w expressions summed over the levels in
// the forward's order, so it is never written to memory.  One CTA owns EMDB_ROWS rows of one direction of one pair;
// each thread keeps its EMDB_Q rows' coordinates and ten ratios in registers and walks the other cloud (coordinates
// and ten ratio rows: 56 B per point, 112 KB at 2048 points -> two CTAs per SM) in shared memory in index order.
// Every sum runs in a fixed order: the result is bit-reproducible.
constexpr int EMDB_THREADS = 256;
constexpr int EMDB_Q = 2;                     // rows per thread
constexpr int EMDB_ROWS = EMDB_THREADS * EMDB_Q;

__host__ __device__ constexpr size_t emdb_smem(int cols) { return (size_t)cols * (sizeof(float4) + EMD_LEVELS * sizeof(float)); }

// grid (pairs, 2 directions, row blocks): direction 0 -> rows are points of xyz1 (grad1), 1 -> points of xyz2 (grad2)
__global__ void __launch_bounds__(EMDB_THREADS, 2)
k_emd_backward(const float* __restrict__ xyz1, const float* __restrict__ xyz2, const float* __restrict__ ratios,
               const float* __restrict__ grad_cost, float* __restrict__ grad1, float* __restrict__ grad2, int n, int m) {
  extern __shared__ float4 smb[];
  __shared__ float slevel[EMD_LEVELS];
  const int p = blockIdx.x, dir = blockIdx.y, tid = threadIdx.x;
  const int nrow = dir ? m : n, ncol = dir ? n : m;
  const int row0 = blockIdx.z * EMDB_ROWS;
  if (row0 >= nrow) return;                              // the shorter direction needs fewer row blocks
  const float* rows = dir ? xyz2 + (size_t)p * m * 3 : xyz1 + (size_t)p * n * 3;
  const float* cols = dir ? xyz1 + (size_t)p * n * 3 : xyz2 + (size_t)p * m * 3;
  const float* rat = ratios + (size_t)p * EMD_LEVELS * (n + m);
  const int roff = dir ? n : 0, coff = dir ? 0 : n;     // ratioL_t at [t][0..n), ratioR_t at [t][n..n+m)
  float4* cxyz = smb;                                    // [ncol]
  float* crat = reinterpret_cast<float*>(cxyz + ncol);   // [EMD_LEVELS][ncol]
  for (int c = tid; c < ncol; c += EMDB_THREADS) cxyz[c] = make_float4(cols[c * 3], cols[c * 3 + 1], cols[c * 3 + 2], 0.f);
  for (int t = 0; t < EMD_LEVELS; ++t)
    for (int c = tid; c < ncol; c += EMDB_THREADS) crat[t * ncol + c] = rat[(size_t)t * (n + m) + coff + c];
  // the forward's levels, evaluated by the same (run-time) powf
  if (tid < EMD_LEVELS) slevel[tid] = tid == EMD_LEVELS - 1 ? 0.0f : -powf(4.0f, 7 - tid);
  float x[EMDB_Q], y[EMDB_Q], z[EMDB_Q], rr[EMDB_Q][EMD_LEVELS], gx[EMDB_Q], gy[EMDB_Q], gz[EMDB_Q];
#pragma unroll
  for (int u = 0; u < EMDB_Q; ++u) {
    const int r = row0 + u * EMDB_THREADS + tid;
    const bool ok = r < nrow;
    x[u] = ok ? rows[r * 3] : 0.f; y[u] = ok ? rows[r * 3 + 1] : 0.f; z[u] = ok ? rows[r * 3 + 2] : 0.f;
#pragma unroll
    for (int t = 0; t < EMD_LEVELS; ++t) rr[u][t] = ok ? rat[(size_t)t * (n + m) + roff + r] : 0.f;
    gx[u] = gy[u] = gz[u] = 0.0f;
  }
  __syncthreads();
  float level[EMD_LEVELS];
#pragma unroll
  for (int t = 0; t < EMD_LEVELS; ++t) level[t] = slevel[t];
  for (int c = 0; c < ncol; ++c) {
    const float4 q = cxyz[c];
    float cr[EMD_LEVELS];
#pragma unroll
    for (int t = 0; t < EMD_LEVELS; ++t) cr[t] = crat[t * ncol + c];
#pragma unroll
    for (int u = 0; u < EMDB_Q; ++u) {
      // d2 and w exactly as k_emd_approx pass 3: emd_d2(xyz1_k, xyz2_l), exp(level d2) * ratioL_k * ratioR_l
      const float d2 = dir ? emd_d2(q.x, q.y, q.z, x[u], y[u], z[u]) : emd_d2(x[u], y[u], z[u], q.x, q.y, q.z);
      float match = 0.0f;
#pragma unroll
      for (int t = 0; t < EMD_LEVELS; ++t) {
        const float w = dir ? __expf(level[t] * d2) * cr[t] * rr[u][t] : __expf(level[t] * d2) * rr[u][t] * cr[t];
        match += w;
      }
      const float d = match * 2;
      gx[u] += (x[u] - q.x) * d;
      gy[u] += (y[u] - q.y) * d;
      gz[u] += (z[u] - q.z) * d;
    }
  }
  const float gc = grad_cost[p];
  float* g = dir ? grad2 + (size_t)p * m * 3 : grad1 + (size_t)p * n * 3;
#pragma unroll
  for (int u = 0; u < EMDB_Q; ++u) {
    const int r = row0 + u * EMDB_THREADS + tid;
    if (r < nrow) { g[r * 3] = gx[u] * gc; g[r * 3 + 1] = gy[u] * gc; g[r * 3 + 2] = gz[u] * gc; }
  }
}

// =====================================================================================
// Chamfer backward (reference: chamfer3D.cu:155-195, NmDistanceGradKernel launched once per direction with fp32
// atomicAdd scatters into zeroed gradients).  Here every output element is owned by one thread and written once:
// for a point i of cloud 1
//   grad1[i] = g_i (x1_i - x2_idx1[i])  then, in ascending j,  + (-(g'_j (x2_j - x1_i)))  for every j with idx2[j] == i
// (g = 2 graddist1, g' = 2 graddist2); cloud 2 symmetrically, but its scattered terms first and its direct term last,
// which is the reference's launch order.  The j are found by scanning the other cloud's index array, staged in shared
// memory in chunks (integer compares only).  Products and sums are rounded one by one (no contraction), as the
// reference's atomics do: an element with at most one scattered term equals the reference's result bit for bit, and
// every element is bit-reproducible.
// =====================================================================================
constexpr int CDB_THREADS = 256;
constexpr int CDB_CHUNK = 4096;               // other-cloud indices staged per pass (16 KB)

__device__ __forceinline__ void cdb_add(float& sx, float& sy, float& sz, float g, float ax, float ay, float az, float bx,
                                        float by, float bz, bool neg) {
  float tx = __fmul_rn(g, __fsub_rn(ax, bx)), ty = __fmul_rn(g, __fsub_rn(ay, by)), tz = __fmul_rn(g, __fsub_rn(az, bz));
  if (neg) { tx = -tx; ty = -ty; tz = -tz; }
  sx = __fadd_rn(sx, tx); sy = __fadd_rn(sy, ty); sz = __fadd_rn(sz, tz);
}

// grid (cdiv(n, T) + cdiv(m, T), B): the first cdiv(n, T) blocks own points of xyz1, the rest points of xyz2
__global__ void __launch_bounds__(CDB_THREADS)
k_chamfer_backward(const float* __restrict__ xyz1, const float* __restrict__ xyz2, const int* __restrict__ idx1,
                   const int* __restrict__ idx2, const float* __restrict__ gd1, const float* __restrict__ gd2,
                   float* __restrict__ gx1, float* __restrict__ gx2, int n, int m) {
  __shared__ int4 sidx[CDB_CHUNK / 4];
  const size_t b = blockIdx.y;
  const int nb1 = (n + CDB_THREADS - 1) / CDB_THREADS;
  const bool two = (int)blockIdx.x >= nb1;              // rows are points of xyz2
  const int na = two ? m : n, nb = two ? n : m;
  const float* A = (two ? xyz2 : xyz1) + b * na * 3;
  const float* Bp = (two ? xyz1 : xyz2) + b * nb * 3;
  const int* ia = (two ? idx2 : idx1) + b * na;
  const int* ib = (two ? idx1 : idx2) + b * nb;
  const float* ga = (two ? gd2 : gd1) + b * na;
  const float* gb = (two ? gd1 : gd2) + b * nb;
  const int i = ((int)blockIdx.x - (two ? nb1 : 0)) * CDB_THREADS + threadIdx.x;
  const bool valid = i < na;
  float ax = 0.f, ay = 0.f, az = 0.f, sx = 0.f, sy = 0.f, sz = 0.f;
  if (valid) {
    ax = A[i * 3]; ay = A[i * 3 + 1]; az = A[i * 3 + 2];
    if (!two) {                                        // cloud 1: direct term first
      const int j = ia[i];
      cdb_add(sx, sy, sz, ga[i] * 2, ax, ay, az, Bp[j * 3], Bp[j * 3 + 1], Bp[j * 3 + 2], false);
    }
  }
  int* s = reinterpret_cast<int*>(sidx);
  for (int c0 = 0; c0 < nb; c0 += CDB_CHUNK) {
    const int cn = min(CDB_CHUNK, nb - c0), cn4 = (cn + 3) >> 2;
    __syncthreads();
    for (int k = threadIdx.x; k < cn4 * 4; k += CDB_THREADS) s[k] = k < cn ? ib[c0 + k] : -1;
    __syncthreads();
    if (!valid) continue;
#pragma unroll 4
    for (int k4 = 0; k4 < cn4; ++k4) {
      const int4 v = sidx[k4];
      if (v.x == i || v.y == i || v.z == i || v.w == i) {
        const int e[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (e[u] != i) continue;
          const int j = c0 + k4 * 4 + u;
          cdb_add(sx, sy, sz, gb[j] * 2, Bp[j * 3], Bp[j * 3 + 1], Bp[j * 3 + 2], ax, ay, az, true);
        }
      }
    }
  }
  if (!valid) return;
  if (two) {                                           // cloud 2: direct term last
    const int j = ia[i];
    cdb_add(sx, sy, sz, ga[i] * 2, ax, ay, az, Bp[j * 3], Bp[j * 3 + 1], Bp[j * 3 + 2], false);
  }
  float* out = (two ? gx2 : gx1) + b * na * 3;
  out[i * 3] = sx; out[i * 3 + 1] = sy; out[i * 3 + 2] = sz;
}

}  // namespace lion

extern "C" int lion_chamfer_backward(const float* xyz1, const float* xyz2, const int* idx1, const int* idx2,
                                     const float* graddist1, const float* graddist2, float* gradxyz1, float* gradxyz2,
                                     int B, int N, int M, void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && idx1 && idx2 && graddist1 && graddist2 && gradxyz1 && gradxyz2 && B > 0 && N > 0 && M > 0,
               "lion_chamfer_backward: bad arguments");
  LION_REQUIRE(B <= 65535, "lion_chamfer_backward: at most 65535 cloud pairs per call (got %d)", B);
  Ctx c;
  c.stream = (cudaStream_t)stream;
  LION_LAUNCH(&c, k_chamfer_backward, dim3(cdiv(N, CDB_THREADS) + cdiv(M, CDB_THREADS), B), CDB_THREADS, 0, xyz1, xyz2, idx1,
              idx2, graddist1, graddist2, gradxyz1, gradxyz2, N, M);
  return check_launch(&c, "lion_chamfer_backward");
}

template <bool SAVE>
static int emd_launch(const float* a, const float* b, float* out, float* ratios, int pairs, int n, int m, int nb, int pairwise,
                      void* stream) {
  Ctx c;
  c.stream = (cudaStream_t)stream;
  const size_t smem = (size_t)EMD_MAX * (2 * sizeof(float4) + 3 * sizeof(float)) + EMD_THREADS * sizeof(float);
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_emd_approx<SAVE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}
  LION_LAUNCH(&c, k_emd_approx<SAVE>, pairs, EMD_THREADS, smem, a, b, out, ratios, n, m, nb, pairwise);
  return check_launch(&c, SAVE ? "lion_emd_approx_saved" : "lion_emd_approx");
}

extern "C" int lion_emd_approx(const float* xyz1, const float* xyz2, float* cost, int B, int N, int M, void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && cost && B > 0 && N > 0 && M > 0, "lion_emd_approx: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_approx: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  return emd_launch<false>(xyz1, xyz2, cost, nullptr, B, N, M, 1, 0, stream);
}

extern "C" int lion_emd_approx_saved(const float* xyz1, const float* xyz2, float* cost, float* ratios, int B, int N, int M,
                                     void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && cost && ratios && B > 0 && N > 0 && M > 0, "lion_emd_approx_saved: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_approx_saved: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  return emd_launch<true>(xyz1, xyz2, cost, ratios, B, N, M, 1, 0, stream);
}

extern "C" int lion_emd_backward(const float* xyz1, const float* xyz2, const float* ratios, const float* grad_cost, float* grad1,
                                 float* grad2, int B, int N, int M, void* stream) {
  LION_REQUIRE(xyz1 && xyz2 && ratios && grad_cost && grad1 && grad2 && B > 0 && N > 0 && M > 0, "lion_emd_backward: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_backward: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  Ctx c;
  c.stream = (cudaStream_t)stream;
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_emd_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)emdb_smem(EMD_MAX)));
  }
  LION_LAUNCH(&c, k_emd_backward, dim3(B, 2, cdiv(N > M ? N : M, EMDB_ROWS)), EMDB_THREADS, emdb_smem(N > M ? N : M), xyz1, xyz2,
              ratios, grad_cost, grad1, grad2, N, M);
  return check_launch(&c, "lion_emd_backward");
}

extern "C" int lion_emd_pairwise(const float* samples, const float* refs, float* out, int n_sample, int n_ref, int N, int M,
                                 void* stream) {
  LION_REQUIRE(samples && refs && out && n_sample > 0 && n_ref > 0 && N > 0 && M > 0, "lion_emd_pairwise: bad arguments");
  LION_REQUIRE(N <= EMD_MAX && M <= EMD_MAX, "lion_emd_pairwise: clouds of at most %d points (got %d, %d)", EMD_MAX, N, M);
  LION_REQUIRE((long long)n_sample * n_ref < (1LL << 31), "lion_emd_pairwise: too many pairs");
  return emd_launch<false>(samples, refs, out, nullptr, n_sample * n_ref, N, M, n_ref, 1, stream);
}

// =====================================================================================
// occupancy grid of the JSD score (reference: utils/evaluation_metrics_fast.py:604-647,
// entropy_of_occupancy_grid: sklearn NearestNeighbors over the grid cells, then per-point Python loops).
//
// One CTA per cloud.  Every thread keeps OCC_Q points in registers as doubles and scans the cell table, staged in
// shared memory as double SoA in chunks of OCC_CHUNK cells, in index order with a strict `<`: the lowest cell index
// wins an exact tie.  The squared distance is the exact float64 one, rounded op by op (no contraction), so the nearest
// cell does not depend on the compiler.  A point adds 1 to point_counts[cell] and sets the cell's bit in the cloud's
// bitmap in shared memory (K bits); once the whole cloud is done, every set bit adds 1 to cloud_counts[cell].  Integer
// atomics only: the counts do not depend on the order the atomics land in.
// =====================================================================================
namespace lion {

constexpr int OCC_THREADS = 256;
constexpr int OCC_Q = 4;                        // points per thread and pass
constexpr int OCC_CHUNK = 1024;                 // cells staged per pass (24 KB of doubles)
constexpr int OCC_BITMAP_MAX = 192 * 1024;      // dynamic shared memory of the bitmap: K <= 1,572,864 cells

__device__ __forceinline__ double occ_d2(double px, double py, double pz, double cx, double cy, double cz) {
  const double dx = __dsub_rn(px, cx), dy = __dsub_rn(py, cy), dz = __dsub_rn(pz, cz);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void __launch_bounds__(OCC_THREADS)
k_occupancy(const float* __restrict__ clouds, const float* __restrict__ cells, int n, int k_cells,
            int* __restrict__ point_counts, int* __restrict__ cloud_counts) {
  __shared__ double sx[OCC_CHUNK], sy[OCC_CHUNK], sz[OCC_CHUNK];
  extern __shared__ unsigned bitmap[];           // [cdiv(k_cells, 32)]
  const int words = (k_cells + 31) >> 5;
  for (int w = threadIdx.x; w < words; w += OCC_THREADS) bitmap[w] = 0u;
  const float* pc = clouds + (size_t)blockIdx.x * n * 3;
  for (int p0 = 0; p0 < n; p0 += OCC_THREADS * OCC_Q) {
    double px[OCC_Q], py[OCC_Q], pz[OCC_Q], best[OCC_Q];
    int bi[OCC_Q];
#pragma unroll
    for (int u = 0; u < OCC_Q; ++u) {
      const int j = p0 + u * OCC_THREADS + threadIdx.x;
      const int jj = j < n ? j : 0;
      px[u] = pc[jj * 3]; py[u] = pc[jj * 3 + 1]; pz[u] = pc[jj * 3 + 2];
      best[u] = CUDART_INF; bi[u] = 0;
    }
    for (int k0 = 0; k0 < k_cells; k0 += OCC_CHUNK) {
      const int kn = min(OCC_CHUNK, k_cells - k0);
      __syncthreads();
      for (int k = threadIdx.x; k < kn; k += OCC_THREADS) {
        sx[k] = cells[(size_t)(k0 + k) * 3]; sy[k] = cells[(size_t)(k0 + k) * 3 + 1]; sz[k] = cells[(size_t)(k0 + k) * 3 + 2];
      }
      __syncthreads();
#pragma unroll 2
      for (int k = 0; k < kn; ++k) {
        const double cx = sx[k], cy = sy[k], cz = sz[k];
#pragma unroll
        for (int u = 0; u < OCC_Q; ++u) {
          const double d = occ_d2(px[u], py[u], pz[u], cx, cy, cz);
          if (d < best[u]) { best[u] = d; bi[u] = k0 + k; }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < OCC_Q; ++u) {
      if (p0 + u * OCC_THREADS + threadIdx.x < n) {
        atomicAdd(point_counts + bi[u], 1);
        atomicOr(bitmap + (bi[u] >> 5), 1u << (bi[u] & 31));
      }
    }
  }
  __syncthreads();
  for (int w = threadIdx.x; w < words; w += OCC_THREADS) {
    unsigned bits = bitmap[w];
    while (bits) {
      const int b = __ffs(bits) - 1;
      bits &= bits - 1;
      atomicAdd(cloud_counts + (w << 5) + b, 1);
    }
  }
}

}  // namespace lion

extern "C" int lion_occupancy_grid(const float* clouds, const float* cells, int S, int N, int K, int* point_counts,
                                   int* cloud_counts, void* stream) {
  LION_REQUIRE(clouds && cells && point_counts && cloud_counts && S > 0 && N > 0 && K > 0, "lion_occupancy_grid: bad arguments");
  LION_REQUIRE((long long)S * N <= INT_MAX, "lion_occupancy_grid: S * N = %lld points exceed INT_MAX", (long long)S * N);
  const size_t bitmap = (size_t)cdiv(K, 32) * sizeof(unsigned);
  LION_REQUIRE(bitmap <= (size_t)OCC_BITMAP_MAX, "lion_occupancy_grid: at most %d cells (got %d)", OCC_BITMAP_MAX * 8, K);
  Ctx c;
  c.stream = (cudaStream_t)stream;
  static DevOnce attr_once;
  if (attr_once.need()) {
    LION_CHECK_CUDA(cudaFuncSetAttribute(k_occupancy, cudaFuncAttributeMaxDynamicSharedMemorySize, OCC_BITMAP_MAX));
  }
  LION_TRY(memset_async(&c, point_counts, 0, (size_t)K * sizeof(int)));
  LION_TRY(memset_async(&c, cloud_counts, 0, (size_t)K * sizeof(int)));
  LION_LAUNCH(&c, k_occupancy, S, OCC_THREADS, bitmap, clouds, cells, N, K, point_counts, cloud_counts);
  return check_launch(&c, "lion_occupancy_grid");
}
